"""The device loader's line parser (graph_b200/csrc/edgelist_scan.h) against the host reader's parse_line
(graph_b200/csrc/edgelist_line.h), compiled with g++ and run on the CPU: an adversarial corpus (empty lines,
CRLF, missing columns, garbage suffixes, 21-digit ids, '+', 1e50, subnormals, inf/nan, hex, incomplete
exponents, float midpoints and their neighbours) and 10^7 random tokens.  Every value the fast path accepts
must be bit-equal to the host's; it may decline, but on printed float32 values less than 1 % of the time."""
import subprocess
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def test_scan_line_matches_parse_line(tmp_path):
    exe = tmp_path / "edgelist_scan_check"
    cmd = ["g++", "-std=c++17", "-O2", "-Wall", "-Wextra", "-Werror", f"-I{ROOT / 'graph_b200' / 'csrc'}",
           str(ROOT / "tests" / "cpp" / "edgelist_scan_check.cpp"), "-o", str(exe)]
    subprocess.run(cmd, check=True, capture_output=True, text=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "edgelist_scan ok" in r.stdout, r.stdout + r.stderr
