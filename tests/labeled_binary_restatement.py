"""A Python restatement of the reference's binary file of a node-labelled graph, written from its Rust source for
the tests: the file of tests/binary_restatement.py with the NodeValues payload in front of the CSRs.

    NodeValues::serialize            crates/builder/src/graph/csr.rs:334-341   [usize n][NV x n]
    DirectedCsrGraph (de)serialize   csr.rs:606-641   NodeValues, csr_out, csr_inc
    UndirectedCsrGraph (de)serialize csr.rs:810-851   NodeValues, csr

NV = u32 takes 4 bytes, u64 / usize 8; the file does not say which, so the reader is told.
"""
import numpy as np

import binary_restatement as br

LABELS = [7, 0, 0xFFFFFFFF, 3]  # the labelled goldens' NodeValues: 0 and 2^32 - 1 included


def write(csrs, name="u32", labels=(), label_bytes=4) -> bytes:
    """csrs as br.write takes them; labels: the NodeValues, label_bytes each (their number is written as the
    count, which may differ from the CSRs' node_count)."""
    head = np.array([len(labels)], "<u8").tobytes() + np.asarray(labels).astype(f"<u{label_bytes}").tobytes()
    return head + br.write(csrs, name)[8:]


def read(data: bytes, ncsr: int, values: bool, label_bytes: int):
    """(labels as u64, br.read's list of CSRs); asserts on anything malformed"""
    assert len(data) >= 8, "unexpected end of file"
    nv = int(np.frombuffer(data[:8], "<u8")[0])
    payload = data[8:8 + nv * label_bytes]
    assert len(payload) == nv * label_bytes, "unexpected end of file"
    labels = np.frombuffer(payload, f"<u{label_bytes}").astype(np.uint64)
    return labels, br.read(data[:8] + data[8 + nv * label_bytes:], ncsr, values)


def labeled_golden_files():
    """name -> bytes of the labelled golden files: the graphs of br.golden_files() with LABELS as their NodeValues,
    as DirectedCsrGraph<u32, u32> / <usize, usize> (and the undirected twins) write them, so u32 files hold 4-byte
    labels and usize files 8-byte labels.  Each is its unlabelled golden with the labels after the count."""
    files = {}
    for name, data in br.golden_files().items():
        label_bytes = br.ID_BYTES["usize" if "_usize" in name else "u32"]
        assert data[:8] == np.array([len(LABELS)], "<u8").tobytes()
        files[name.replace("binary_", "binary_labeled_", 1)] = (data[:8] + np.array(LABELS, f"<u{label_bytes}").tobytes()
                                                                + data[8:])
    return files
