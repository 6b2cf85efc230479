"""A Python restatement of the reference's binary graph file, written from its Rust source for the tests:
a writer and a reader over numpy CSR arrays.

    NodeValues::serialize            crates/builder/src/graph/csr.rs:334-341   [usize n] (NV = (): no payload)
    Csr::serialize / deserialize     csr.rs:252-313   [usize L][type name][NI n][NI entries][NI offsets x (n+1)]
                                                      [Target<NI, EV> x entries]
    DirectedCsrGraph (de)serialize   csr.rs:606-626   NodeValues, csr_out, csr_inc
    UndirectedCsrGraph (de)serialize csr.rs:817-824   NodeValues, csr

Little-endian, usize = 8 bytes; Target<NI, EV> is #[repr(C)] (graph/mod.rs:6-10): (u32, f32) 8 bytes,
(u64, f32) 16 bytes with 4 bytes of padding (written as zero here).
"""
import numpy as np

ID_BYTES = {"u32": 4, "u64": 8, "usize": 8}
EDGES = [(0, 1), (0, 2), (1, 2), (1, 3), (2, 3), (3, 1)]  # the graph of the reference's serialize tests


def record_dtype(name: str, values: bool) -> np.dtype:
    it = f"<u{ID_BYTES[name]}"
    if not values:
        return np.dtype(it)
    fields = [("target", it), ("value", "<f4")]
    if ID_BYTES[name] == 8:
        fields.append(("pad", "<u4"))
    return np.dtype(fields)


def csr_bytes(off, tgt, val=None, name="u32") -> bytes:
    it = np.dtype(f"<u{ID_BYTES[name]}")
    off = np.asarray(off)
    rec = np.zeros(len(tgt), record_dtype(name, val is not None))
    if val is None:
        rec[:] = tgt
    else:
        rec["target"] = tgt
        rec["value"] = val
    return b"".join([np.array([len(name)], "<u8").tobytes(), name.encode(),
                     np.array([len(off) - 1, len(tgt)], it).tobytes(), off.astype(it).tobytes(), rec.tobytes()])


def write(csrs, name="u32") -> bytes:
    """csrs: [(offsets, targets, values or None)] — directed: [csr_out, csr_inc]; undirected: [csr]."""
    n = len(csrs[0][0]) - 1
    return np.array([n], "<u8").tobytes() + b"".join(csr_bytes(o, t, v, name) for o, t, v in csrs)


def read(data: bytes, ncsr: int, values: bool):
    """[(offsets, targets, values or None)] as u64 / f32 arrays; asserts on anything malformed."""
    pos = 0

    def take(k):
        nonlocal pos
        b = data[pos:pos + k]
        assert len(b) == k, "unexpected end of file"
        pos += k
        return b

    nv = int(np.frombuffer(take(8), "<u8")[0])
    out = []
    for _ in range(ncsr):
        name = take(int(np.frombuffer(take(8), "<u8")[0])).decode()
        it = f"<u{ID_BYTES[name]}"
        n, e = (int(x) for x in np.frombuffer(take(2 * ID_BYTES[name]), it))
        assert n == nv, "number of node values must be the same as node count"
        off = np.frombuffer(take((n + 1) * ID_BYTES[name]), it).astype(np.uint64)
        dt = record_dtype(name, values)
        rec = np.frombuffer(take(e * dt.itemsize), dt)
        if values:
            out.append((off, rec["target"].astype(np.uint64), rec["value"].copy()))
        else:
            out.append((off, rec.astype(np.uint64), None))
    assert pos == len(data), "trailing bytes"
    return out


def in_values(out_off, out_tgt, out_w, in_off, in_tgt):
    """The in-CSR values a weighted digraph is written with: the k-th occurrence of s in in-row t gets the
    value of the k-th occurrence of t in out-row s."""
    w = np.empty(len(in_tgt), np.float32)
    for t in range(len(in_off) - 1):
        seen = {}
        for j in range(int(in_off[t]), int(in_off[t + 1])):
            s = int(in_tgt[j])
            k = seen.get(s, 0)
            seen[s] = k + 1
            row = range(int(out_off[s]), int(out_off[s + 1]))
            hits = [i for i in row if int(out_tgt[i]) == t]
            w[j] = out_w[hits[k]]
    return w


def sorted_csr(edges, n, undirected=False):
    """Sorted CSR (rows ascending, duplicates kept; for undirected both directions) of a small edge list."""
    pairs = list(edges) + ([(d, s) for s, d in edges] if undirected else [])
    pairs.sort()
    off = np.zeros(n + 1, np.uint64)
    for s, _ in pairs:
        off[s + 1] += 1
    return np.cumsum(off).astype(np.uint64), np.array([d for _, d in pairs], np.uint64)


def golden_files():
    """name -> bytes of the golden files: directed and undirected, u32 and usize, with and without values."""
    n = 4
    out_off, out_tgt = sorted_csr(EDGES, n)
    in_off, in_tgt = sorted_csr([(d, s) for s, d in EDGES], n)
    und_off, und_tgt = sorted_csr(EDGES, n, undirected=True)
    value = {e: np.float32(0.5 + i) for i, e in enumerate(EDGES)}
    out_w = np.array([value[(s, int(t))] for s in range(n) for t in out_tgt[out_off[s]:out_off[s + 1]]], np.float32)
    in_w = in_values(out_off, out_tgt, out_w, in_off, in_tgt)
    und_w = np.arange(len(und_tgt), dtype=np.float32) * np.float32(0.25)
    files = {}
    for name in ("u32", "usize"):
        files[f"binary_directed_{name}.bin"] = write([(out_off, out_tgt, None), (in_off, in_tgt, None)], name)
        files[f"binary_directed_{name}_values.bin"] = write([(out_off, out_tgt, out_w), (in_off, in_tgt, in_w)], name)
        files[f"binary_undirected_{name}.bin"] = write([(und_off, und_tgt, None)], name)
        files[f"binary_undirected_{name}_values.bin"] = write([(und_off, und_tgt, und_w)], name)
    return files
