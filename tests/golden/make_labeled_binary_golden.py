#!/usr/bin/env python3
"""Writes the labelled binary graph golden files tests/golden/binary_labeled_*.bin.

The graphs of make_binary_golden.py with NodeValues [7, 0, 2^32 - 1, 3] in front of the CSRs, restated from the
reference's serializer (tests/labeled_binary_restatement.py cites csr.rs:334-341, :606-641, :810-851); they were
not produced by Rust.  The u32 files hold u32 labels and the usize files usize labels, as DirectedCsrGraph<u32, u32>
and DirectedCsrGraph<usize, usize> write them.
"""
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))

from labeled_binary_restatement import labeled_golden_files  # noqa: E402


def main():
    for name, data in labeled_golden_files().items():
        (HERE / name).write_bytes(data)
        print("wrote", HERE / name, len(data), "bytes")


if __name__ == "__main__":
    main()
