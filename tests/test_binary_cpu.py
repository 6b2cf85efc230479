"""The host decoder of binary graph files (gb_binary_decode, graph_b200/csrc/io.cu + binary_format.h) against
the Python restatement of the reference's format (tests/binary_restatement.py), on the CPU: the golden files
decode to the restatement's arrays, and every malformed variant is rejected with a message naming the problem."""
import numpy as np
import pytest

import binary_restatement as br
import graph_b200 as gb

GOLDEN_NAMES = sorted(br.golden_files())


def test_golden_files_are_the_restatement(golden_dir):
    for name, data in br.golden_files().items():
        assert (golden_dir / name).read_bytes() == data, name
    # the first offsets of a u32 directed file start at byte 27 (8 + 8 + 3 + 4 + 4): offsets 0, 2, 4, 5, 6
    raw = (golden_dir / "binary_directed_u32.bin").read_bytes()
    assert raw[19:27] == np.array([4, 6], "<u4").tobytes()
    assert raw[27:47] == np.array([0, 2, 4, 5, 6], "<u4").tobytes()


@pytest.mark.parametrize("name", GOLDEN_NAMES)
def test_decoder_matches_restatement(golden_dir, name):
    data = (golden_dir / name).read_bytes()
    directed = "directed" in name and "undirected" not in name
    values = name.endswith("_values.bin")
    want = br.read(data, 2 if directed else 1, values)
    got = gb._decode_binary(data, directed, with_values=values)
    if directed:
        oo, ot, ow, io, it = got
        assert (oo == want[0][0]).all() and (ot == want[0][1]).all()
        assert (io == want[1][0]).all() and (it == want[1][1]).all()
        if values:
            assert ow.tobytes() == want[0][2].tobytes()
    else:
        off, tgt = got
        assert (off == want[0][0]).all() and (tgt == want[0][1]).all()
    # values are dropped on request, and cannot be asked of a file without them
    gb._decode_binary(data, directed, with_values=False)
    if not values:
        with pytest.raises(ValueError, match="no edge values"):
            gb._decode_binary(data, directed, with_values=True)


def test_u32_and_usize_decode_alike(golden_dir):
    for kind in ("directed", "undirected"):
        for v in ("", "_values"):
            a = gb._decode_binary((golden_dir / f"binary_{kind}_u32{v}.bin").read_bytes(), kind == "directed", bool(v))
            b = gb._decode_binary((golden_dir / f"binary_{kind}_usize{v}.bin").read_bytes(), kind == "directed", bool(v))
            for x, y in zip(a, b, strict=True):
                assert (x is None and y is None) or x.tobytes() == y.tobytes()


def test_file_sizes():
    n, m = 4, len(br.EDGES)
    files = br.golden_files()
    assert len(files["binary_directed_u32.bin"]) == 8 * m + 8 * n + 54  # 8m + 8n + 54
    assert len(files["binary_directed_u32_values.bin"]) == 16 * m + 8 * n + 54


def section_boundaries(data, ncsr, values, name="u32"):
    """byte offsets where a header field or array ends, plus offsets inside the records"""
    w = br.ID_BYTES[name]
    rec = br.record_dtype(name, values).itemsize
    cuts, pos = [8], 8
    for _ in range(ncsr):
        L = int(np.frombuffer(data[pos:pos + 8], "<u8")[0])
        n, e = (int(x) for x in np.frombuffer(data[pos + 8 + L:pos + 8 + L + 2 * w], f"<u{w}"))
        pos += 8
        cuts.append(pos)
        pos += L
        cuts += [pos, pos + w, pos + 2 * w]
        pos += 2 * w + (n + 1) * w
        cuts += [pos - w // 2, pos]
        cuts += [pos + rec // 2, pos + rec, pos + e * rec - 1]
        pos += e * rec
    return sorted(set(c for c in cuts if 0 < c < len(data)))


@pytest.mark.parametrize("name", GOLDEN_NAMES)
def test_truncation_is_rejected(golden_dir, name):
    data = (golden_dir / name).read_bytes()
    directed = "undirected" not in name
    for cut in [0, 1, 7] + section_boundaries(data, 2 if directed else 1, name.endswith("_values.bin"),
                                             "usize" if "usize" in name else "u32"):
        with pytest.raises(ValueError, match="end of file|holds an undirected|neither|trailing"):
            gb._decode_binary(data[:cut], directed)


def test_trailing_bytes_are_rejected(golden_dir):
    for name in GOLDEN_NAMES:
        data = (golden_dir / name).read_bytes()
        directed = "undirected" not in name
        for extra in (b"\0", b"\0" * 4, b"\0" * 64):
            with pytest.raises(ValueError, match="trailing"):
                gb._decode_binary(data + extra, directed)


def directed_csrs():
    n = 4
    o, t = br.sorted_csr(br.EDGES, n)
    i, it = br.sorted_csr([(d, s) for s, d in br.EDGES], n)
    return (o, t), (i, it)


@pytest.mark.parametrize("bad", ["i64", "u16", "u8", "", "x" * 100])
def test_unknown_type_names(bad):
    (o, t), (i, it) = directed_csrs()
    good = br.write([(o, t, None), (i, it, None)])
    data = good[:8] + np.array([len(bad)], "<u8").tobytes() + bad.encode() + good[8 + 8 + 3:]
    with pytest.raises(ValueError, match='invalid id size, expected "u32" bytes, got'):
        gb._decode_binary(data, True)
    # the same name in csr_inc
    head = br.csr_bytes(o, t)
    inc = br.csr_bytes(i, it)
    data = good[:8] + head + np.array([len(bad)], "<u8").tobytes() + bad.encode() + inc[8 + 3:]
    with pytest.raises(ValueError, match="invalid id size|end of file"):
        gb._decode_binary(data, True)


def test_count_mismatches():
    (o, t), (i, it) = directed_csrs()
    # NodeValues count != node_count (lib.rs:295)
    good = br.write([(o, t, None), (i, it, None)])
    with pytest.raises(ValueError, match="number of node values must be the same as node count"):
        gb._decode_binary(np.array([5], "<u8").tobytes() + good[8:], True)
    # csr_inc with another node_count
    i5 = np.append(i, i[-1])
    with pytest.raises(ValueError, match="differ in node_count"):
        gb._decode_binary(br.write([(o, t, None)]) + br.csr_bytes(i5, it), True)
    # csr_inc with other entries
    it2 = np.append(it, 0)
    i2 = i.copy()
    i2[-1] += 1
    with pytest.raises(ValueError, match="differ in entries"):
        gb._decode_binary(br.write([(o, t, None)]) + br.csr_bytes(i2, it2), True)
    # csr_inc with another id type
    with pytest.raises(ValueError, match="differ in id type"):
        gb._decode_binary(br.write([(o, t, None)]) + br.csr_bytes(i, it, name="u64"), True)
    # node_count 0
    with pytest.raises(ValueError, match="node_count must be > 0"):
        gb._decode_binary(br.write([(np.array([0]), np.array([]), None)]), False)


def test_offsets_and_targets_are_checked():
    (o, t), (i, it) = directed_csrs()
    cases = []
    bad = o.copy(); bad[0] = 1; cases.append((bad, t, "offsets\\[0\\] must be 0"))
    bad = o.copy(); bad[1], bad[2] = bad[2], bad[1]; cases.append((bad, t, "not monotone"))
    bad = o.copy(); bad[-1] -= 1; cases.append((bad, t, "offsets end at"))
    bad = t.copy(); bad[0] = 4; cases.append((o, bad, "targets >= node_count"))
    for off, tgt, msg in cases:
        with pytest.raises(ValueError, match=msg):
            gb._decode_binary(br.write([(off, tgt, None), (i, it, None)]), True)
        with pytest.raises(ValueError, match=msg):
            gb._decode_binary(br.write([(i, it, None), (off, tgt, None)]), True)


def test_wrong_kind_says_which_kind():
    (o, t), (i, it) = directed_csrs()
    for values in (None, np.ones(len(t), np.float32)):
        d = br.write([(o, t, values), (i, it, values)])
        with pytest.raises(ValueError, match="holds a directed graph"):
            gb._decode_binary(d, False)
        u = br.write([(o, t, values)])
        with pytest.raises(ValueError, match="holds an undirected graph"):
            gb._decode_binary(u, True)


def test_u64_ids_must_fit_32_bits():
    (o, t), (i, it) = directed_csrs()
    big = t.copy(); big[0] = 1 << 32
    with pytest.raises(ValueError, match="does not fit 32 bits"):
        gb._decode_binary(br.write([(o, big, None), (i, it, None)], "u64"), True)
    off = o.copy(); off[1:] += 1 << 32
    with pytest.raises(ValueError, match="does not fit 32 bits"):
        gb._decode_binary(br.write([(off, t, None), (i, it, None)], "usize"), True)
    # node_count above 32 bits in the header
    data = bytearray(br.write([(o, t, None), (i, it, None)], "u64"))
    data[0:8] = np.array([1 << 32], "<u8").tobytes()
    data[8 + 8 + 3:8 + 8 + 3 + 8] = np.array([1 << 32], "<u8").tobytes()
    with pytest.raises(ValueError, match="does not fit 32 bits"):
        gb._decode_binary(bytes(data), True)


def test_ids_just_below_32_bits_narrow():
    """A u64 file whose ids are all below 2^32 narrows; 2^32 - 1 is a target only of a graph with n = 2^32,
    which does not fit, so the largest id tried here is the largest a small graph can hold."""
    (o, t), (i, it) = directed_csrs()
    got = gb._decode_binary(br.write([(o, t, None), (i, it, None)], "u64"), True)
    assert got[1].tolist() == t.tolist() and got[4].tolist() == it.tolist()


def test_single_node_without_edges(golden_dir):
    z = (np.array([0, 0]), np.array([], np.uint64), None)
    got = gb._decode_binary(br.write([z, z]), True)
    assert got[0].tolist() == [0, 0] and len(got[1]) == 0
    off, tgt = gb._decode_binary(br.write([z], "usize"), False)
    assert off.tolist() == [0, 0] and len(tgt) == 0
