"""CPU: the condensed-KKT kernels' plan and admission rules, restated in tests/cond_plan.py.

* The admitted component counts per component size, dtype and equality rows, over the scene sizes n.
* `comp_apply` covers t < U NT positions of the grid t < cs << sh. With U = 4 for every cs, fp32 scenes of 129-150
  five-row components and of 257-258 three-row components were admitted with their last row slot past the grid's
  1024 positions (the three-row ones only at n = 49-65, where the 16 list entries per column leave room for them only
  when their rows touch one body). Sized per cs, U covers every admitted scene.
* The verdicts of the scenes the GPU tests (tests/test_gpu_cond_limits.py) use, so that a test meant for the
  condensed kernel cannot quietly run on the dual form.
"""
import pytest
import torch

from tests import band_plan as bp
from tests import cond_plan as cp


def _admitted(ts, e, cs, n):
    """Component counts of cs uniform rows admitted at n, with the per-column limit for one-body rows (3 columns)."""
    out = []
    for ncomp in range(1, 4 * cp.NT // cs + 1):
        plan = cp.make_plan(ts, n, ncomp * cs, e)
        if plan is not None and ncomp * cs * cs <= plan["wcap"] and 3 * ncomp <= cp.LMAX * n:
            out.append(ncomp)
    return out


def test_apply_span():
    assert {cs: cp.apply_span(cs) for cs in range(1, 7)} == {1: 4, 2: 4, 3: 6, 4: 4, 5: 5, 6: 6}


def test_plans_of_the_benchmark_shapes():
    # cfg 3 (fp32, 32 bodies, 64 contacts) and cfg 2 (fp64, 16 bodies, 32 contacts x 5 rows): two CTAs per SM
    p3 = cp.make_plan(4, 96, 256, 0)
    assert (p3["NS"], p3["pcap"], p3["wcap"], p3["ctas_per_sm"]) == (6, 256, 1024, 2), p3
    p2 = cp.make_plan(8, 48, 160, 0)
    assert (p2["NS"], p2["ctas_per_sm"]) == (3, 2), p2
    # m > 1024 or n + e > 128: no condensed plan
    assert cp.make_plan(8, 120, 1028, 0) is None and cp.make_plan(4, 126, 64, 3) is None
    # the shared memory binds long before m = 1024: at n = 120 fp32 plans reach m = 704, fp64 plans m = 432
    assert cp.make_plan(4, 120, 704, 0)["mult"] == 4 and cp.make_plan(4, 120, 708, 0) is None
    assert cp.make_plan(8, 120, 432, 0)["mult"] == 4 and cp.make_plan(8, 120, 436, 0) is None
    assert all(cp.make_plan(ts, n, 1024, 0) is None for ts in (4, 8) for n in range(1, 129))
    # cfg 2's formulation on cfg 3's pile: wcap drops from 6 to 5 to 4 pcap as contacts grow, then no plan
    mults = {nc: (lambda p: p and p["mult"])(cp.make_plan(4, 96, 5 * nc, 0)) for nc in (128, 140, 145, 146, 147, 152, 153)}
    assert mults == {128: 6, 140: 6, 145: 5, 146: 5, 147: 4, 152: 4, 153: None}, mults


TABLE_N = list(range(3, 129, 9))


@pytest.mark.parametrize("ts", [4, 8])
def test_admitted_component_counts(ts):
    """The largest admitted count per (e, cs) at each n of TABLE_N, summarised as (smallest, largest) over n."""
    got = {}
    for e in (0, 3):
        for cs in range(1, 7):
            top = [max(_admitted(ts, e, cs, n), default=0) for n in TABLE_N if n + e <= 128]
            got[(e, cs)] = (min(top), max(top))
    want = TABLES[ts]
    assert got == want, got


TABLES = {
    4: {(0, 1): (16, 640), (0, 2): (16, 384), (0, 3): (16, 258), (0, 4): (16, 195), (0, 5): (16, 150), (0, 6): (16, 120),
        (3, 1): (16, 640), (3, 2): (16, 382), (3, 3): (16, 257), (3, 4): (16, 195), (3, 5): (16, 150), (3, 6): (16, 120)},
    8: {(0, 1): (16, 496), (0, 2): (16, 259), (0, 3): (16, 174), (0, 4): (16, 131), (0, 5): (16, 101), (0, 6): (16, 81),
        (3, 1): (16, 496), (3, 2): (16, 257), (3, 3): (16, 173), (3, 4): (16, 130), (3, 5): (16, 101), (3, 6): (16, 81)},
}


def test_old_apply_rule_ranges():
    """Admitted scenes whose grid cs << sh exceeds 4 positions per thread, as (ncomp range, n range) per
    (sizeof(T), e, cs); the fixed rule covers every admitted scene, mixed component sizes included
    (ncomp cs <= pcap <= 4 NT)."""
    found = {}
    for ts in (4, 8):
        for e in (0, 3):
            for cs in range(1, 7):
                for n in range(3, 129 - e):
                    for ncomp in _admitted(ts, e, cs, n):
                        st = dict(cs=cs, sh=cp.ceil_log2(ncomp))
                        assert cp.apply_grid_ok(st), (ts, e, cs, n, ncomp)
                        if not cp.apply_grid_ok(st, old=True):
                            found.setdefault((ts, e, cs), []).append((ncomp, n))
    got = {k: ((min(c for c, _ in v), max(c for c, _ in v)), (min(n for _, n in v), max(n for _, n in v)))
           for k, v in found.items()}
    assert got == {(4, 0, 3): ((257, 258), (49, 65)), (4, 0, 5): ((129, 150), (25, 124)),
                   (4, 3, 3): ((257, 258), (49, 61)), (4, 3, 5): ((129, 150), (25, 98))}, got
    for cs in range(1, 7):
        for ncomp in range(1, 4 * cp.NT // cs + 1):
            assert cp.apply_grid_ok(dict(cs=cs, sh=cp.ceil_log2(ncomp)))


# ------------------------------------------------------------------ verdicts of the GPU tests' scenes
def _verdict(inp, dtype):
    Q, p, G, h, A, b, F = inp
    e = A.shape[1] if A.dim() > 1 else 0
    plan = cp.make_plan(cp.tsize(dtype), Q.shape[1], G.shape[1], e)
    return [cp.verdict_dense(Q[s], G[s], F[s], e, plan) for s in range(Q.shape[0])]


def _one(vs):
    assert all(v == vs[0] for v in vs), vs
    v = vs[0]
    return (v["rule"],) if not v["ok"] else (v["ncomp"], v["cs"], v["sh"], v["band_lu"])


def test_verdicts_of_the_block_count_scenes():
    from tests.test_gpu_cond_limits import NS_SCENES
    got = {}
    for NS, (nb, nc) in NS_SCENES.items():
        for e in (0, 3):
            inp = cp.contact_scenes(1, nb, nc, 2, e=e, seed=40 + NS)
            for dtype in (torch.float32, torch.float64):
                plan = cp.make_plan(cp.tsize(dtype), 3 * nb, 4 * nc, e)
                assert plan["NS"] == NS
                got[(NS, e, cp.tsize(dtype))] = _one(_verdict(inp, dtype))
    assert all(v[:3] == (nc, 4, cp.ceil_log2(nc)) for (NS, e, _), v in got.items()
               for nc in [NS_SCENES[NS][1]]), got
    assert {k: v[3] for k, v in got.items() if k[1] == 0} == BAND_LU, got


BAND_LU = {(NS, 0, ts): True for NS in (2, 3, 4, 6, 8) for ts in (4, 8)}   # pile contacts: narrow band


def test_verdicts_of_the_component_size_scenes():
    from tests.test_gpu_cond_limits import CS_SCENES
    got = {name: _one(_verdict(build(), dtype)) for name, (build, cs) in CS_SCENES.items()
           for dtype in (torch.float64,)}
    assert got == CS_VERDICTS, got


CS_VERDICTS = {"cs1_poststab": (32, 1, 5, True), "cs2_monotone_block": (32, 2, 5, True), "cs3_fd1": (32, 3, 5, True),
               "cs4_fd2": (32, 4, 5, True), "cs5_fd3": (32, 5, 5, True), "cs6_fd4": (32, 6, 5, True),
               "mixed_4_and_1": (33, 4, 6, True)}


def test_verdicts_of_the_limit_scenes():
    got = {}
    for name in cp.LIMIT_SCENES:
        dtype, inside, outside = cp.limit_scenes(name)
        got[name] = (_one(_verdict(inside, dtype)), _one(_verdict(outside, dtype)))
    assert got == LIMIT_VERDICTS, got


LIMIT_VERDICTS = {
    "KS_entries_per_row": ((24, 4, 5, True), ("KS",)),
    "UC_columns_per_component": ((24, 4, 5, True), ("UC",)),
    "CSMAX_rows_per_component": ((24, 6, 5, True), ("CSMAX",)),
    "LMAX_entries_per_column": ((36, 4, 6, False), ("LMAX",)),
    "pcap_padded_positions": ((25, 4, 5, True), ("pcap",)),
    "wcap_after_make_cplan": ((146, 5, 8, False), ("wcap",)),
    "plan_shared_memory": ((108, 4, 7, False), ("plan",)),
}


def test_verdicts_of_the_comp_apply_scenes():
    from lcp_physics_b200.scenes import make_scenes
    v = _one(_verdict(make_scenes(1, 32, 140, fd=3, e=0, dtype=torch.float64, seed=61), torch.float32))
    assert v[:3] == (140, 5, 8), v
    inp = cp.dense_from_graph(cp.floor_contacts(20, 257), 1, 1, seed=62)
    v = _one(_verdict(inp, torch.float32))
    assert v[:3] == (257, 3, 9), v
    # the same scenes in fp64 do not fit the shared memory: the dual form takes them
    assert cp.make_plan(8, 96, 700, 0) is None or _one(_verdict(make_scenes(1, 32, 140, fd=3, dtype=torch.float64,
                                                                            seed=61), torch.float64))[0] == "wcap"


def test_engine_verdicts():
    ok, bad = bp.hubs(1, 16, ring=40), bp.hubs(1, 17, ring=40)
    got = []
    for sc in (ok, bad):
        nc = len(sc["body1"])
        plan = cp.make_plan(8, 3 * sc["nb"], 4 * nc, 0)
        v = cp.verdict_soa(sc["nb"], sc["body1"], sc["body2"], nc, 0, 0, plan)
        got.append(v["rule"] if not v["ok"] else (v["ncomp"], v["cs"], v["sh"]))
    assert got == [(56, 4, 6), "LMAX"], got
    for ts, nc in ((8, 108), (4, 176)):
        sc = cp.circulant(40, nc)
        plan = cp.make_plan(ts, 120, 4 * nc, 0)
        assert [(lambda v: (v["ncomp"], v["sh"]))(cp.verdict_soa(40, sc["body1"], sc["body2"], nc, 0, 0, plan, count=k))
                for k in (0, 1, nc)] == [(0, 0), (1, 0), (nc, cp.ceil_log2(nc))]
        assert cp.verdict_soa(40, sc["body1"], sc["body2"], nc, 0, 0, plan, count=nc + 1)["rule"] == "count"
        assert cp.make_plan(ts, 120, 4 * nc + 4, 0) is None
    for nb in (36, 40):
        assert cp.make_plan(4, 3 * nb, 8 * nb, 0)["NS"] == 8 and cp.make_plan(8, 3 * nb, 8 * nb, 0)["NS"] == 8
