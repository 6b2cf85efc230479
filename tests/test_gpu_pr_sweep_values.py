"""Single JACOBI PageRank sweeps from integer-valued source vectors, checked bit for bit (helpers in
tests/pr_sweep_values.py).  The ranks-after-many-sweeps tests start from init / outdeg, where tied neighbours of
the internal order hold the same value, so a gather from the wrong source can pass them unseen
(tests/test_pr_sweep_values_model.py shows the difference on the CPU).

Every case drives gb_pr_shard_step from vectors it chooses, on sweeps 1, 2 and 3:
  * x_cur holds random integers on the sources the shard's rows gather and a NaN naming the source on every
    other one, so that every row sum is exact in any order and reading a source no row gathers writes a NaN;
  * every owned active row of scores and x_next must equal pr_update restated in numpy f32, byte for byte;
  * scores and x_next start as a sentinel NaN (scores hold known old values on the owned rows): only the owned
    active rows change; with peer stores every peer's x_next receives exactly the owner's rows; x_cur is
    unchanged, except that sweep 1 writes base / outdeg into its rows without in-edges;
  * the error share is the sum of |score - old| over the owned rows, plus rank 0's closed form on sweep 1;
  * with virtual blocks, every slot of the value buffer V that the layout model gives a pair holds its source's
    value, and pass A writes nothing but the runs and their pads.
The internal order is read back through gb_pr_shard_finish and must be the layout model's, and each case asserts
the plan shape or statistics that name its path."""
import ctypes as C

import numpy as np
import pytest

import pr_path_fixtures as fx
import pr_sweep_values as sv
import test_gpu_pr_fused_pass_a as fp
import test_gpu_pr_vsectors as vs
import vblock_fixtures as vf

pytestmark = pytest.mark.gpu

lm = fx.lm
SHAPE_KEYS = ("hot_blocks", "n_cb", "n_fin", "n_fin_warp", "fin_u", "grid_fin", "fin_hub_ctas", "n_mega", "dual",
              "last_hot_block")
VB_KEYS = ("vblock_parts", "vblock_pairs", "vblock_edges")
SWEEPS = (1, 2, 3)
SMALL_WINDOW = vs.SMALL_WINDOW
VB = {"GB_PR_VBLOCKS": 1}
MEGA = 200   # GB_PR_MEGA of the small-chunk case, as test_page_rank_column_block_knobs


def knob_id(env):
    return "-".join(f"{k[6:]}={v}" for k, v in env.items()) or "defaults"


# (graph, knobs, the path check): "path" = the plan shape of the layout model, and fx.check_path at the defaults;
# "vb" = the virtual blocks with the model's counts, slots, tasks and V map; "sell" = no virtual blocks, SELL runs
CASES = (
    [(name, {}, "path") for name in fx.FIXTURES]
    + [(name, dict(VB), "vb") for name in vf.VB_FIXTURES]
    + [(name, {**VB, "GB_PR_VB_WINDOW": SMALL_WINDOW}, "vb") for name in ("rmat18", "tail_r1", "few_active")]
    + [("equal_degrees", {**VB, "GB_PR_TAU": 0}, "vb"),
       ("equal_degrees", {**VB, "GB_PR_TAU": 0, "GB_PR_VB_WINDOW": SMALL_WINDOW}, "vb"),
       ("star_in", {**VB, "GB_PR_TAU": 0}, "sell"),
       ("rmat18", {"GB_PR_TAU": 0}, "path")]
    + [(name, {"GB_PR_VBLOCKS": 2}, "sell") for name in ("rmat18", "repeated_source", "tail_r33")]
    + [(name, {"GB_PR_CHUNK": 32, "GB_PR_MEGA": MEGA}, "path") for name in ("rmat18", "repeated_source", "star_in")]
    + [("rmat18", {"GB_PR_CHUNK": 512, "GB_PR_TASK_CHUNKS": 64}, "path"),
       ("rmat18", {"GB_PR_TASK_CHUNKS": 128}, "path")]
    + [("rmat18", env, "path") for env in ({"GB_PR_FIN_U": 4}, {"GB_PR_FIN_SPLIT": 1},
                                           {"GB_PR_FIN_U": 4, "GB_PR_FIN_SPLIT": 1}, {"GB_PR_FIN_SPLIT": 2})]
    + [("capped_finish", env, "path") for env in ({"GB_PR_FIN_U": 2}, {"GB_PR_FIN_U": 2, "GB_PR_FIN_SPLIT": 1},
                                                  {"GB_PR_FIN_SPLIT": 1})]
    + [("rmat22", {}, "path"), ("rmat22", dict(VB), "vb")])
# virtual-rank shards of one device: every rank with the host exchange and with peer stores
SHARD_CASES = [("rmat18", {}, "path"), ("rmat18", dict(VB), "vb"), ("few_active", {}, "path"),
               ("repeated_source", {}, "path"), ("equal_degrees", {**VB, "GB_PR_TAU": 0}, "vb")]


@pytest.fixture(scope="module")
def gb():
    import graph_b200
    return graph_b200


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


_RMAT22: dict = {}


def graph(gb, name):
    """(n, out CSR, in CSR) of a path fixture, or of RMAT-22 (seed 42, Sorted) as the device builds it"""
    if name != "rmat22":
        _, _, n, out, inc = fx.graph(name)
        return n, out, inc
    if not _RMAT22:
        g = gb.DiGraph.rmat(22, seed=42, layout=gb.Layout.Sorted)
        _RMAT22["csr"] = (g.node_count(), tuple(a.copy() for a in g.csr("out")),
                          tuple(a.copy() for a in g.csr("in")))
    return _RMAT22["csr"]


def set_knobs(monkeypatch, name, env):
    for k in ("GB_PR_VBLOCKS", "GB_PR_VB_WINDOW"):
        monkeypatch.delenv(k, raising=False)
    fx.set_knobs(monkeypatch, name, **env)


def plan_model(gb, name, env, P=1, p=0):
    n, out, inc = graph(gb, name)
    B = lm.clamp_block((fx.FIXTURES[name][1] if name in fx.FIXTURES else None) or lm.CB_BLOCK_DEFAULT)
    tau = 1e30 if env.get("GB_PR_TAU") == 0 else lm.CB_TAU_DEFAULT
    return lm.make_plan(inc[0].astype(np.int64), inc[1], np.diff(out[0].astype(np.int64)), B, tau, P=P, p=p,
                        mega=env.get("GB_PR_MEGA", lm.CB_MEGA_DEG))


def assert_path(gb, b, name, env, kind, sms, P, p):
    """the shard's plan took the path the case names; returns the layout model's V map of pass A (or None)"""
    n, out, inc = graph(gb, name)
    plan = plan_model(gb, name, env, P, p)
    shape, info = b.plan_shape(), b.stats
    assert info["active_rows"] == plan["n_active"] and info["local_rows"] == plan["n_loc"]
    if kind == "vb":
        assert info["vblock_parts"] > 0 and shape["grid_sell"] == 0, info
        assert {k: info[k] for k in VB_KEYS} == lm.vb_counts(plan, inc[0], inc[1])
        if name not in fx.FIXTURES or P > 1:   # the full model's layout build is a Python loop over the rows
            return None
        tau = env.get("GB_PR_TAU")
        m = vs.model(name, tau, P, p, env.get("GB_PR_VB_WINDOW", lm.VB_WINDOW))
        vs.assert_stats(info, m)
        if "GB_PR_VB_WINDOW" not in env:
            fp.assert_counts(info, fp.fused_model(name, tau, P, p))
        return m
    assert info["vblock_parts"] == 0
    fin = dict(fin_u=env.get("GB_PR_FIN_U", 0), fin_split=env.get("GB_PR_FIN_SPLIT", 0))
    want = lm.launch_shape(plan, sms=sms, **fin)
    assert {k: shape[k] for k in SHAPE_KEYS} == {k: want[k] for k in SHAPE_KEYS}, (name, env)
    assert {k: info[k] for k in ("segments", "groups", "block_edges")} == lm.layout_counts(plan, inc[0], inc[1])
    if kind == "sell":
        assert shape["grid_sell"] > 0
    if "GB_PR_MEGA" in env:
        assert shape["n_mega"] > 0 and info["cut_segments"] > 0, (shape, info)   # sort path, segments cut by chunks
    elif "GB_PR_TASK_CHUNKS" in env and "GB_PR_CHUNK" not in env:
        assert info["chunk_groups"] != 512
    if P == 1 and not env and name in fx.FIXTURES and sms == lm.H100_SMS:
        fx.check_path(name, plan, {**want, **shape})
    if "GB_PR_FIN_SPLIT" in env and env["GB_PR_FIN_SPLIT"] == 1:
        assert shape["fin_hub_ctas"] > 0
    return None


def bits(t):
    return t.cpu().numpy().view(np.uint32)


def same_bits(got, want, what):
    """got == want byte for byte (uint32 views); on a mismatch: how many, and the first with both values"""
    bad = np.flatnonzero(got != want)
    if len(bad):
        i = int(bad[0])
        f = lambda u: (hex(int(u)), float(np.uint32(u).view(np.float32)))
        raise AssertionError(f"{what}: {len(bad)} entries differ, first {i}: got {f(got[i])}, want {f(want[i])}")


def check_internal_order(b, ic):
    """gb_pr_shard_finish of arange(n) reads back new_id: the layout model's order"""
    import torch
    n = ic["n"]
    got = b.finish(torch.arange(n, dtype=torch.float32, device=b.device)).cpu().numpy()
    assert (got.astype(np.int64) == ic["new_id"]).all(), "the plan's internal order is the layout model's"


def check_sweeps(b, P, p, ic, peers, m=None):
    """sweeps 1, 2, 3 of rank p of P from its own integer vectors, each checked bit for bit (see the module doc);
    with peers, the step stores into P - 1 peer vectors; m: the layout model's V map of pass A, checked too"""
    import torch
    from graph_b200._capi import check, lib
    n, na = ic["n"], ic["n_active"]
    assert b.n_active == na
    dev = b.device
    sentinel = np.full(n, sv.SENTINEL, np.uint32)
    dev_of = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.float32)).to(dev)
    mine = sv.owned(n, na, P, p)
    used = sv.gathered(ic, mine)
    b.init(sv.DAMPING, *(torch.empty(n, dtype=torch.float32, device=dev) for _ in range(3)))
    for sweep_no in SWEEPS:
        what = (P, p, sweep_no, "peers" if peers else "host")
        x = sv.vector(ic, used, 100 * P + 10 * p + sweep_no)
        old = (np.random.default_rng(sweep_no).random(n) * 1000).astype(np.float32)
        score, xn = sv.expected(ic, x)
        x_cur = dev_of(x)
        nxt = [dev_of(sentinel) for _ in range(P if peers else 1)]   # this rank's, then its peers'
        sc = dev_of(np.where(mine, old.view(np.uint32), sentinel))
        err = torch.full((1,), float("nan"), dtype=torch.float64, device=dev)
        ptrs = [t.data_ptr() for t in nxt[1:]] if peers and P > 1 else None
        if m is not None:
            torch.cuda.synchronize()
            check(lib.gb_pr_shard_plan_values(b._shard, 1, None, m["slots"]))
        b.step(sv.DAMPING, sweep_no, x_cur, nxt[0], ptrs, sc, err)
        torch.cuda.synchronize()
        same_bits(bits(sc), np.where(mine, score.view(np.uint32), sentinel), f"scores {what}")
        want_xn = np.where(mine, xn.view(np.uint32), sentinel)
        for q, t in enumerate(nxt):
            same_bits(bits(t), want_xn, f"x_next of {'this rank' if q == 0 else f'peer {q}'} {what}")
        want_x = x.copy()
        if sweep_no == 1:
            want_x[na:] = sv.fill_inactive(ic)
        same_bits(bits(x_cur), want_x.view(np.uint32), f"x_cur {what}")
        e = sv.error_share(ic, score, old, mine, sweep_no, p)
        assert abs(err.item() - e) <= 1e-12 * abs(e), (what, err.item(), e)
        if m is not None:
            check_values(b, m, x, what)


def check_values(b, m, x, what):
    """pass A wrote every pair's slot with its source's value, the pad slots with +0.0, and nothing else"""
    from graph_b200._capi import check, lib
    V = np.empty(m["slots"], np.float32)
    check(lib.gb_pr_shard_plan_values(b._shard, 0, V.ctypes.data_as(C.c_void_p), m["slots"]))
    got, pair, pad = V.view(np.uint32), m["V"] >= 0, m["V"] == -2
    same_bits(got[pair], x[m["V"][pair]].view(np.uint32), f"V slots of the pairs {what}")
    assert (got[pad] == 0).all(), ("pad slots are +0.0", what)
    assert (got[~pair & ~pad] == 0xFFFFFFFF).all(), ("pass A writes nothing outside the runs and pads", what)


def run_case(gb, monkeypatch, sms, name, env, kind, P, peers_modes, backends=None):
    from graph_b200.multigpu import CudaShardBackend
    set_knobs(monkeypatch, name, env)
    n, out, inc = graph(gb, name)
    if backends is None:
        g = gb.DiGraph.from_csr(out[0], out[1], inc[0], inc[1])
        backends = [CudaShardBackend(g, p, P) for p in range(P)]
    ic = sv.internal(plan_model(gb, name, env), out, inc)
    check_internal_order(backends[0], ic)
    models = [assert_path(gb, b, name, env, kind, sms, P, p) for p, b in enumerate(backends)]
    for peers in peers_modes:
        for p, b in enumerate(backends):
            check_sweeps(b, P, p, ic, peers, models[p])


@pytest.mark.parametrize("name,env,kind", CASES, ids=[f"{c[0]}-{knob_id(c[1])}" for c in CASES])
def test_one_rank_sweeps_bit_exact(gb, monkeypatch, sms, name, env, kind):
    run_case(gb, monkeypatch, sms, name, env, kind, 1, (False,))


@pytest.mark.parametrize("world", [2, 5])
@pytest.mark.parametrize("name,env,kind", SHARD_CASES, ids=[f"{c[0]}-{knob_id(c[1])}" for c in SHARD_CASES])
def test_virtual_rank_sweeps_bit_exact(gb, monkeypatch, sms, name, env, kind, world):
    run_case(gb, monkeypatch, sms, name, env, kind, world, (False, True))


@pytest.mark.parametrize("env,kind", [({}, "path"), (dict(VB), "vb")], ids=["defaults", "VBLOCKS=1"])
@pytest.mark.parametrize("v", [2, 3])
def test_streamed_csr_shards_sweeps_bit_exact(gb, monkeypatch, sms, v, env, kind):
    """the shards of gb_pr_shards_csr_u32 (the streamed host-CSR layout build), v ranks on one device"""
    name = "rmat18"
    set_knobs(monkeypatch, name, env)
    n, out, inc = graph(gb, name)
    backends = gb.Comm([0]).pr_shards_csr(inc[0], inc[1], out[0], ranks_per_device=v)
    run_case(gb, monkeypatch, sms, name, env, kind, v, (False, True), backends)
