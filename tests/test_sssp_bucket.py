"""The delta-stepping bucket advance (graph_b200/csrc/sssp_bucket.h) on the CPU: compiled with g++ and run over
delta from 1e-45 (subnormal) to 1e30 and distances from 0 to FLT_MAX.  Before it had its own bounded
function, a delta of 1e-20 or below made the host loop of sssp.cu spin forever."""
import subprocess
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def test_bucket_advance_is_bounded_and_holds_dmin(tmp_path):
    exe = tmp_path / "sssp_bucket_check"
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", f"-I{ROOT / 'graph_b200' / 'csrc'}",
           str(ROOT / "tests" / "cpp" / "sssp_bucket_check.cpp"), "-o", str(exe)]
    subprocess.run(cmd, check=True, capture_output=True, text=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "sssp_bucket ok" in r.stdout, r.stdout + r.stderr
