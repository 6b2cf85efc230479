#!/usr/bin/env python3
"""Writes the binary graph golden files tests/golden/binary_*.bin.

The bytes are restated from the reference's serializer (tests/binary_restatement.py cites csr.rs:252-341,
:606-626, :817-824) for the graph of its serialize tests (csr.rs:1046-1167:
(0,1),(0,2),(1,2),(1,3),(2,3),(3,1)); they were not produced by Rust.  Directed and undirected, NI = u32 and
usize, with and without f32 values (value of edge i = i + 0.5; undirected entry j = j / 4).
"""
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))

from binary_restatement import golden_files  # noqa: E402


def main():
    for name, data in golden_files().items():
        (HERE / name).write_bytes(data)
        print("wrote", HERE / name, len(data), "bytes")


if __name__ == "__main__":
    main()
