"""The host decoder of labelled binary graph files (gb_binary_decode_labeled, graph_b200/csrc/io.cu +
binary_format.h) against the Python restatement of the reference's format (tests/labeled_binary_restatement.py),
on the CPU: the labelled goldens decode to the restatement's labels and CSRs, and every malformed variant is
rejected with a message naming the problem.  A labelled file is [usize n][NV x n] followed by the CSRs; NV's width is not in the
file, so the caller gives it."""
import numpy as np
import pytest

import binary_restatement as br
import labeled_binary_restatement as lbr
import graph_b200 as gb

LABELED = lbr.labeled_golden_files()
NAMES = sorted(LABELED)
EOF_MESSAGE = "binary graph file: unexpected end of file"


def shape(name):
    """(directed, values, label_bytes) of a golden file name"""
    directed = "undirected" not in name
    return directed, name.endswith("_values.bin"), 8 if "_usize" in name else 4


def directed_csrs():
    n = 4
    o, t = br.sorted_csr(br.EDGES, n)
    i, it = br.sorted_csr([(d, s) for s, d in br.EDGES], n)
    return [(o, t, None), (i, it, None)]


def test_labeled_goldens_are_the_restatement(golden_dir):
    assert len(NAMES) == 8
    for name, data in LABELED.items():
        assert (golden_dir / name).read_bytes() == data, name
        directed, values, label_bytes = shape(name)
        labels, csrs = lbr.read(data, 2 if directed else 1, values, label_bytes=label_bytes)
        assert labels.tolist() == lbr.LABELS
        # write() with labels gives the same bytes
        id_name = "usize" if label_bytes == 8 else "u32"
        assert lbr.write(csrs, id_name, labels=labels, label_bytes=label_bytes) == data, name
    # the labelled files are not among the unlabelled goldens
    assert not set(LABELED) & set(br.golden_files())
    # u32 directed: [4][7, 0, 2^32 - 1, 3], then csr_out's header at byte 24
    raw = (golden_dir / "binary_labeled_directed_u32.bin").read_bytes()
    assert raw[:24] == np.array([4], "<u8").tobytes() + np.array(lbr.LABELS, "<u4").tobytes()
    assert raw[24:35] == np.array([3], "<u8").tobytes() + b"u32"


@pytest.mark.parametrize("name", NAMES)
def test_decoder_matches_restatement(golden_dir, name):
    data = (golden_dir / name).read_bytes()
    directed, values, label_bytes = shape(name)
    labels, want = lbr.read(data, 2 if directed else 1, values, label_bytes=label_bytes)
    got = gb._decode_binary_labeled(data, directed, label_bytes, with_values=values)
    assert got[0].dtype == np.uint32 and got[0].tolist() == labels.tolist()
    if directed:
        _, oo, ot, ow, io, it = got
        assert (oo == want[0][0]).all() and (ot == want[0][1]).all()
        assert (io == want[1][0]).all() and (it == want[1][1]).all()
        if values:
            assert ow.tobytes() == want[0][2].tobytes()
    else:
        _, off, tgt = got
        assert (off == want[0][0]).all() and (tgt == want[0][1]).all()
    # values are dropped on request, and cannot be asked of a file without them
    dropped = gb._decode_binary_labeled(data, directed, label_bytes, with_values=False)
    if directed:
        assert dropped[3] is None
    if not values:
        with pytest.raises(ValueError, match="no edge values"):
            gb._decode_binary_labeled(data, directed, label_bytes, with_values=True)
    # the CSRs are those of the unlabelled golden
    plain = gb._decode_binary((golden_dir / name.replace("binary_labeled_", "binary_")).read_bytes(), directed)
    for x, y in zip(got[1:] if not directed else (got[1], got[2], got[4], got[5]),
                    plain if not directed else (plain[0], plain[1], plain[3], plain[4]), strict=True):
        assert x.tobytes() == y.tobytes()


def test_u32_and_usize_decode_alike(golden_dir):
    for kind in ("directed", "undirected"):
        for v in ("", "_values"):
            a = gb._decode_binary_labeled((golden_dir / f"binary_labeled_{kind}_u32{v}.bin").read_bytes(),
                                          kind == "directed", 4, bool(v))
            b = gb._decode_binary_labeled((golden_dir / f"binary_labeled_{kind}_usize{v}.bin").read_bytes(),
                                          kind == "directed", 8, bool(v))
            for x, y in zip(a, b, strict=True):
                assert (x is None and y is None) or x.tobytes() == y.tobytes()


@pytest.mark.parametrize("name", NAMES)
def test_every_truncation_is_rejected(name):
    """Every prefix fails with the end-of-file message, except where the format's own ambiguities make the prefix
    look like a whole file of another shape, as they do for unlabelled files: a directed file cut after csr_out
    holds an undirected graph, and since the file does not state the record size, an undirected file with values
    cut between the two record-size ends ends "neither with 4- nor with 8-byte records (unexpected end of file
    ...)", and cut exactly at the size without values it is read as one and its targets fail the CSR checks."""
    data = LABELED[name]
    directed, values, label_bytes = shape(name)
    id_name = "usize" if label_bytes == 8 else "u32"  # NI = NV in the goldens
    rec = br.record_dtype(id_name, True).itemsize - br.ID_BYTES[id_name]  # bytes a record's value adds
    plain_end = len(data) - 2 * len(br.EDGES) * rec  # the size of the file without values (2m entries)
    for cut in range(len(data)):
        with pytest.raises(ValueError) as e:
            gb._decode_binary_labeled(data[:cut], directed, label_bytes)
        msg = str(e.value)
        if msg == EOF_MESSAGE:
            continue
        if directed:
            assert msg == "binary graph file holds an undirected graph, not a directed one", (cut, msg)
        else:
            assert values and cut >= plain_end, (cut, msg)
            assert ("unexpected end of file" in msg) == (cut > plain_end), (cut, msg)


def test_truncation_right_after_csr_out_reads_as_undirected():
    """The one cut of a directed file that is not an end of file: what is left is a whole undirected file."""
    data = LABELED["binary_labeled_directed_u32.bin"]
    csr_inc = br.csr_bytes(*directed_csrs()[1][:2])
    with pytest.raises(ValueError, match="holds an undirected graph"):
        gb._decode_binary_labeled(data[:len(data) - len(csr_inc)], True, 4)


@pytest.mark.parametrize("label_bytes", [4, 8])
def test_count_mismatch(label_bytes):
    csrs = directed_csrs()
    for labels in ([1, 2, 3], [1, 2, 3, 4, 5]):
        data = lbr.write(csrs, labels=labels, label_bytes=label_bytes)
        with pytest.raises(ValueError, match="^number of node values must be the same as node count$"):
            gb._decode_binary_labeled(data, True, label_bytes)


@pytest.mark.parametrize("label_bytes", [4, 8])
def test_absurd_count_is_an_end_of_file(label_bytes):
    """A count of 2^63 (or any that the file cannot hold) places nothing and sizes nothing."""
    good = lbr.write(directed_csrs(), labels=lbr.LABELS, label_bytes=label_bytes)
    for count in (1 << 63, (1 << 64) - 1, (1 << 61) + 1, len(good)):
        data = np.array([count], "<u8").tobytes() + good[8:]
        with pytest.raises(ValueError, match=f"^{EOF_MESSAGE}$"):
            gb._decode_binary_labeled(data, True, label_bytes)


def test_wide_label_names_the_smallest_node():
    csrs = directed_csrs()
    for labels, node in (([1, 2, 1 << 32, (1 << 64) - 1], 2), ([1, 2, 1 << 32, 3], 2), ([1, 2, 3, 1 << 40], 3),
                         ([(1 << 32) + 5, 0, 0, 0], 0)):
        for directed, c in ((True, csrs), (False, [br.sorted_csr(br.EDGES, 4, undirected=True) + (None,)])):
            data = lbr.write(c, "usize", labels=np.array(labels, np.uint64), label_bytes=8)
            with pytest.raises(ValueError, match=f"^binary graph file: the node value of node {node} does not fit 32 bits$"):
                gb._decode_binary_labeled(data, directed, 8)
    # 2^32 - 1 is the largest label that narrows
    data = lbr.write(csrs, "usize", labels=np.array([0xFFFFFFFF] * 4, np.uint64), label_bytes=8)
    assert gb._decode_binary_labeled(data, True, 8)[0].tolist() == [0xFFFFFFFF] * 4


@pytest.mark.parametrize("label_bytes", [0, 2, 16, 1, 3, 5])
def test_label_bytes_must_be_4_or_8(label_bytes):
    data = LABELED["binary_labeled_directed_u32.bin"]
    with pytest.raises(ValueError, match=f"^label_bytes must be 4 \\(NV = u32\\) or 8 \\(NV = u64 / usize\\), not {label_bytes}$"):
        gb._decode_binary_labeled(data, True, label_bytes)


@pytest.mark.parametrize("label_bytes", [4, 8])
def test_unlabeled_goldens_fail_under_the_labeled_decoder(golden_dir, label_bytes):
    for name in br.golden_files():
        data = (golden_dir / name).read_bytes()
        with pytest.raises(ValueError):
            gb._decode_binary_labeled(data, "undirected" not in name, label_bytes)


def test_labeled_goldens_fail_under_the_unlabeled_decoder(golden_dir):
    for name in NAMES:
        data = (golden_dir / name).read_bytes()
        with pytest.raises(ValueError):
            gb._decode_binary(data, "undirected" not in name)


@pytest.mark.parametrize("name", NAMES)
def test_wrong_width_is_rejected(name):
    """A file read with the other NV width places its first CSR header elsewhere and fails."""
    directed, _, label_bytes = shape(name)
    with pytest.raises(ValueError):
        gb._decode_binary_labeled(LABELED[name], directed, 12 - label_bytes)


def test_csr_checks_still_apply():
    (o, t, _), (i, it, _) = directed_csrs()
    bad = t.copy()
    bad[0] = 4
    with pytest.raises(ValueError, match="targets >= node_count"):
        gb._decode_binary_labeled(lbr.write([(o, bad, None), (i, it, None)], labels=lbr.LABELS), True, 4)
    with pytest.raises(ValueError, match="trailing"):
        gb._decode_binary_labeled(LABELED["binary_labeled_directed_u32.bin"] + b"\0", True, 4)
    with pytest.raises(ValueError, match="holds a directed graph"):
        gb._decode_binary_labeled(LABELED["binary_labeled_directed_u32.bin"], False, 4)
    # a wide label is reported before the CSRs' problems: the labels come first in the file
    data = lbr.write([(o, bad, None), (i, it, None)], "usize", labels=np.array([0, 1 << 33, 0, 0], np.uint64),
                    label_bytes=8)
    with pytest.raises(ValueError, match="node value of node 1"):
        gb._decode_binary_labeled(data, True, 8)


def test_single_node_without_edges():
    z = (np.array([0, 0]), np.array([], np.uint64), None)
    for label_bytes in (4, 8):
        got = gb._decode_binary_labeled(lbr.write([z, z], labels=[9], label_bytes=label_bytes), True, label_bytes)
        assert got[0].tolist() == [9] and got[1].tolist() == [0, 0] and len(got[2]) == 0


def test_load_labeled_argument_checks(golden_dir):
    for cls in (gb.DiGraph, gb.Graph):
        with pytest.raises(ValueError, match="label_bytes"):
            cls.load_labeled(golden_dir / "test.graph", label_bytes=8)
        for fmt in (gb.FileFormat.Graph500, gb.FileFormat.EdgeList):
            with pytest.raises(ValueError, match="DotGraph or Binary"):
                cls.load_labeled(golden_dir / "test.el", file_format=fmt)


def test_graph_mate_exposes_the_labeled_binary_calls():
    import graph_mate
    for cls in (graph_mate.DiGraph, graph_mate.Graph):
        assert cls.load_labeled is getattr(gb, cls.__name__).load_labeled
        assert hasattr(cls, "serialize_labeled")
    assert graph_mate.FileFormat.Binary is gb.FileFormat.Binary
