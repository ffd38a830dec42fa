"""CPU: the dual-form kernels' plan and per-scene branches, restated in tests/dual_plan.py.

* Every tier boundary in both dtypes: the threads per CTA, T's residency as m grows at several n, the exact windows
  of the split plan, each of the four residencies of G and Q^-1, and where staging G in T's region stops.
* Invariants at every planned shape: the shared memory fits the opt-in limit, the split plan's lower part and its
  tiles fit, the workspace regions are disjoint and ws_per_cta covers them.
* The plan and the per-scene verdicts of every shape tests/test_gpu_dual_limits.py uses, so that a change to the plan
  that moves a GPU test out of its intended tier fails here.
"""
import pytest
import torch

from tests import dual_plan as dp


def _first(ts, n, e, pred, lo=1, hi=1200):
    """Smallest m in [lo, hi) whose plan satisfies pred."""
    return next((m for m in range(lo, hi) if dp.make_plan(ts, n, m, e) and pred(dp.make_plan(ts, n, m, e))), None)


def _window(ts, n, e, pred, hi=1200):
    ms = [m for m in range(1, hi) if dp.make_plan(ts, n, m, e) and pred(dp.make_plan(ts, n, m, e))]
    return (ms[0], ms[-1]) if ms else None


def test_threads_per_cta():
    for ts, nb in ((4, 32), (8, 16)):
        assert dp.make_plan(ts, 24, 1, 0)["nt"] == 128
        assert _first(ts, 24, 0, lambda p: p["nt"] == 256) == 64 - nb + 1       # mp >= 64
        assert _first(ts, 24, 0, lambda p: p["nt"] == 512) == 96 - nb + 1       # mp >= 96
        assert dp.make_plan(ts, 96, 1, 0)["nt"] == 512                          # n >= 96
        assert dp.make_plan(ts, 95, 1, 0)["nt"] == 128


def test_residency_of_t():
    """mode 0 -> 1 -> 2 as m grows; the split plan exists only in narrow windows."""
    got = {(ts, n): (_window(ts, n, 0, lambda p: p["mode"] == 0), _window(ts, n, 0, lambda p: p["mode"] == 1),
                     _first(ts, n, 0, lambda p: p["mode"] == 2)) for ts in (4, 8) for n in (12, 48, 96, 150)}
    assert got == {
        (4, 12): ((1, 224), (225, 256), 257), (4, 48): ((1, 224), (225, 256), 257),
        (4, 96): ((1, 192), (193, 256), 257), (4, 150): ((1, 192), (193, 256), 257),
        (8, 12): ((1, 144), (145, 160), 161), (8, 48): ((1, 144), (145, 160), 161),
        (8, 96): ((1, 144), (145, 160), 161), (8, 150): ((1, 144), (145, 160), 161)}, got


def test_split_windows():
    """fp32: mp = 224 or 256 (m1 = 128); fp64: mp = 160 only (m1 = 80). The uneven split (n2 < m1) and the padded
    split (mp > m) the GPU tests use."""
    for ts, n in ((4, 96), (8, 48), (8, 96)):
        for m in range(1, 1200):
            p = dp.make_plan(ts, n, m, 0)
            if p and p["mode"] == 1:
                assert (p["mp"], p["m1"]) in (((224, 128), (256, 128)) if ts == 4 else ((160, 80),)), (ts, n, m, p)
    p = dp.make_plan(4, 96, 200, 0)
    assert (p["mode"], p["mp"], p["m1"], p["n2"]) == (1, 224, 128, 96)
    p = dp.make_plan(8, 48, 148, 0)
    assert (p["mode"], p["mp"], p["m1"], p["n2"]) == (1, 160, 80, 80)


def test_residency_of_g_and_qinv():
    """Each of the four combinations, per mode, with the m window at the n quoted."""
    win = lambda ts, n, mode, G, Qi: _window(ts, n, 0, lambda p: (p["mode"], p["G_smem"], p["Qi_smem"]) == (mode, G, Qi))
    assert win(8, 48, 0, False, True) == (129, 144)           # G in L2, Q^-1 in shared memory, T in shared memory
    assert win(8, 96, 2, True, False) == (161, 237)           # G in shared memory, Q^-1 in L2, T in L2
    assert win(8, 96, 0, False, False) == (113, 144)
    assert win(8, 48, 2, False, True) == (433, 1199)
    assert win(8, 150, 2, False, False) == (225, 1199)
    assert win(4, 96, 1, False, False) == (193, 256)
    assert win(4, 96, 2, True, True) == (257, 411)
    assert win(4, 96, 2, False, True) == (496, 1199)


def test_staging_of_g():
    """G is staged in T's region when m ldG fits m1 ldT (modes 0 and 1); never in mode 2. More dofs than rows: no."""
    assert dp.make_plan(8, 96, 40, 0)["stage_ld"] == 0
    assert dp.make_plan(8, 96, 96, 0)["stage_ld"] > 0
    assert dp.make_plan(4, 96, 44, 0)["stage_ld"] == 0 and dp.make_plan(4, 96, 36, 0)["stage_ld"] > 0
    assert all(dp.make_plan(ts, n, m, 0)["stage_ld"] == 0 for ts in (4, 8) for n in (12, 96) for m in (300, 600))
    assert _first(8, 96, 0, lambda p: p["stage_ld"] > 0, lo=3) == 65


@pytest.mark.parametrize("optin", [dp.H100_SMEM_OPTIN, 101376, 166912])
@pytest.mark.parametrize("ts", [4, 8])
def test_invariants(ts, optin):
    for n in list(range(3, 160, 7)) + [96, 150]:
        for e in (0, 3):
            for m in list(range(1, 300)) + list(range(300, 1100, 13)):
                p = dp.make_plan(ts, n, m, e, optin)
                if p is None:
                    continue
                assert p["smem_bytes"] <= optin - 1024, (ts, n, m, e, p)
                assert p["mp"] % dp.blk(ts) == 0 and p["mp"] >= m
                if p["mode"] == 1:
                    assert 0 < p["n2"] <= p["m1"] and p["tiles"] <= p["nt"] // 32 and p["m1"] % dp.blk(ts) == 0
                if p["mode"] != 2:
                    assert p["ldT"] >= p["mp"] and p["ldT"] * ts % 16 == 0
                    if p["stage_ld"]:
                        assert m * p["stage_ld"] <= p["m1"] * p["ldT"] and p["stage_ld"] >= n
                end = 0
                for name, (off, size) in p["regions"].items():
                    assert off == end and off % 4 == 0 and size >= 0, (name, p["regions"])
                    end = off + size
                assert end == p["ws_per_cta"]
                r = p["regions"]
                assert r["R"][1] >= m * m and r["Fell"][1] >= 8 * m and r["Gell"][1] >= 16 * m + 64 * n
                assert r["T"][1] >= (p["mp"] * p["ldT"] if p["mode"] == 2 else 0)
                assert r["U12"][1] >= (p["m1"] * p["n2"] if p["mode"] == 1 else 0)


def test_describe_format():
    p = dp.make_plan(4, 96, 256, 0)
    assert dp.describe(p) == ("dual: threads=512 smem=%dB T:smem-split(U12 in L2) m1=128 ldT=260 ldL=132 G:L2 Qinv:L2"
                              % p["smem_bytes"])


def test_verdicts():
    inp = dp.engine_scenes(2, 16, 24, 2, seed=1)
    p = dp.make_plan(8, 48, 96, 0)
    v = dp.verdict(inp[0][0], inp[2][0], inp[6][0], p)
    assert v == dict(qdiag=True, singular=False, rform="staged", f_ell=True, g_ell="n/a", prefetch=True, overlap=True)
    assert dp.verdict(dp.nondiag_q(inp)[0][0], inp[2][0], inp[6][0], p)["rform"] == "gemm"
    assert dp.verdict(dp.singular_q(inp, [0])[0][0], inp[2][0], inp[6][0], p)["singular"]
    # the saved R of scene k of the host pipeline sits at k m^2 elements: aligned for even m
    assert not dp.verdict(inp[0][0], inp[2][0], inp[6][0], p, r_aligned=False)["prefetch"]
    # F^T under the exact adjoint: the engine's gamma columns hold fd + 1 = 3 entries
    assert dp.verdict(inp[0][0], inp[2][0], inp[6][0], p, transF=True)["f_ell"]


def _v(inp, plan):
    vs = dp.verdicts(inp, plan)
    assert all(x == vs[0] for x in vs), vs
    x = vs[0]
    return (x["rform"], x["f_ell"], x["g_ell"], x["prefetch"], x["overlap"])


def test_pins_of_the_tier_shapes():
    from tests.test_gpu_dual_limits import TIERS, build_tier
    got = {}
    for name in TIERS:
        for e in (0, 3):
            dtype, inp = build_tier(name, e, 2)
            p = dp.make_plan(4 if dtype == torch.float32 else 8, *dp.sizes(inp))
            got[(name, e)] = (dp.tier(p)[:4] + (p["mp"], p["m1"]), _v(inp, p))
    assert got == TIER_PINS, got


def test_pins_of_the_ell_shapes():
    from tests.test_gpu_dual_limits import ELL_CASES, ELL_SHAPES, build_ell
    got = {}
    for shape in ELL_SHAPES:
        for which, k in ELL_CASES:
            inp = build_ell(shape, which, k)
            v = _v(inp, dp.make_plan(8, *dp.sizes(inp)))
            got[(shape, which, k)] = (v[1], v[2])
    assert got == ELL_PINS, got


def test_pins_of_the_multi_scene_shapes():
    """mp != m at every shape (the padded tails are in play); the kinds take the branches they are named for."""
    from tests.test_gpu_dual_limits import MULTI_SHAPES, multi_kinds, multi_order
    for shape, (dtype, nb, nc) in MULTI_SHAPES.items():
        p = dp.make_plan(4 if dtype == torch.float32 else 8, 3 * nb, 4 * nc, 0)
        assert p["mp"] != p["m"] and p["mode"] == {"m0": 0, "split": 1, "m2": 2}[shape.split("_")[1]], (shape, p)
        kinds = multi_kinds(nb, nc)
        v = {k: dp.verdicts(x, p)[0] for k, x in kinds.items()}
        assert v["singular_q"]["singular"] and not any(v[k]["singular"] for k in v if k != "singular_q")
        assert v["nondiag_q"]["rform"] == "gemm" and v["diag"]["rform"] in ("staged", "unstaged")
        assert not v["dense_F"]["f_ell"] and v["diag"]["f_ell"]
        if not p["G_smem"]:
            assert v["dense_G"]["g_ell"] is False and v["diag"]["g_ell"] is True
        assert bool(torch.isnan(kinds["nonfinite_h"][3]).any())
    for grid in (132, 264):
        order = multi_order(grid, 6)
        pairs = {(order[c], order[c + grid]) for c in range(grid)}
        assert len(order) == 2 * grid + 3 and len(pairs) == 36


TIER_PINS = {
    ('f64_m0_nt128', 0): ((128, 0, 'smem', 'smem', 32, 32), ('staged', True, 'n/a', True, True)),
    ('f64_m0_nt128', 3): ((128, 0, 'smem', 'smem', 32, 32), ('staged', True, 'n/a', True, True)),
    ('f64_m0_nt256', 0): ((256, 0, 'smem', 'smem', 64, 64), ('staged', True, 'n/a', True, False)),
    ('f64_m0_nt256', 3): ((256, 0, 'smem', 'smem', 64, 64), ('staged', True, 'n/a', True, False)),
    ('f64_m0_nt512', 0): ((512, 0, 'smem', 'smem', 96, 96), ('staged', True, 'n/a', True, True)),
    ('f64_m0_nt512', 3): ((512, 0, 'smem', 'smem', 96, 96), ('staged', True, 'n/a', True, True)),
    ('f64_m0_unstaged', 0): ((512, 0, 'smem', 'smem', 48, 48), ('unstaged', True, 'n/a', True, False)),
    ('f64_m0_unstaged', 3): ((512, 0, 'smem', 'smem', 48, 48), ('unstaged', True, 'n/a', True, False)),
    ('f64_m0_G_L2', 0): ((512, 0, 'L2', 'smem', 144, 144), ('staged', True, True, True, False)),
    ('f64_m0_G_L2', 3): ((512, 0, 'L2', 'smem', 144, 144), ('staged', True, True, True, False)),
    ('f64_m0_G_L2_Qi_L2', 0): ((512, 0, 'L2', 'L2', 144, 144), ('staged', True, True, True, False)),
    ('f64_m0_G_L2_Qi_L2', 3): ((512, 0, 'L2', 'L2', 144, 144), ('staged', True, True, True, False)),
    ('f64_split_even', 0): ((512, 1, 'L2', 'smem', 160, 80), ('staged', True, True, True, True)),
    ('f64_split_even', 3): ((512, 1, 'L2', 'smem', 160, 80), ('staged', True, True, True, True)),
    ('f64_split_padded', 0): ((512, 1, 'L2', 'smem', 160, 80), ('staged', True, True, True, False)),
    ('f64_split_padded', 3): ((512, 1, 'L2', 'smem', 160, 80), ('staged', True, True, True, False)),
    ('f64_m2', 0): ((512, 2, 'smem', 'smem', 176, 176), ('unstaged', True, 'n/a', False, False)),
    ('f64_m2', 3): ((512, 2, 'smem', 'smem', 176, 176), ('unstaged', True, 'n/a', False, False)),
    ('f64_m2_Qi_L2', 0): ((512, 2, 'smem', 'L2', 208, 208), ('unstaged', True, 'n/a', False, False)),
    ('f64_m2_Qi_L2', 3): ((512, 2, 'smem', 'L2', 208, 208), ('unstaged', True, 'n/a', False, False)),
    ('f64_m2_G_L2', 0): ((512, 2, 'L2', 'smem', 208, 208), ('unstaged', True, True, False, False)),
    ('f64_m2_G_L2', 3): ((512, 2, 'L2', 'smem', 208, 208), ('unstaged', True, True, False, False)),
    ('f64_m2_G_L2_Qi_L2', 0): ((512, 2, 'L2', 'L2', 240, 240), ('unstaged', True, True, False, False)),
    ('f64_m2_G_L2_Qi_L2', 3): ((512, 2, 'L2', 'L2', 240, 240), ('unstaged', True, True, False, False)),
    ('f32_m0_nt128', 0): ((128, 0, 'smem', 'smem', 32, 32), ('staged', True, 'n/a', True, True)),
    ('f32_m0_nt128', 3): ((128, 0, 'smem', 'smem', 32, 32), ('staged', True, 'n/a', True, True)),
    ('f32_m0_nt256', 0): ((256, 0, 'smem', 'smem', 64, 64), ('staged', True, 'n/a', True, False)),
    ('f32_m0_nt256', 3): ((256, 0, 'smem', 'smem', 64, 64), ('staged', True, 'n/a', True, False)),
    ('f32_m0_nt512', 0): ((512, 0, 'smem', 'smem', 96, 96), ('staged', True, 'n/a', True, True)),
    ('f32_m0_nt512', 3): ((512, 0, 'smem', 'smem', 96, 96), ('staged', True, 'n/a', True, True)),
    ('f32_m0_G_L2', 0): ((512, 0, 'L2', 'smem', 192, 192), ('staged', True, True, True, False)),
    ('f32_m0_G_L2', 3): ((512, 0, 'L2', 'smem', 192, 192), ('staged', True, True, True, False)),
    ('f32_split_even', 0): ((512, 1, 'L2', 'L2', 256, 128), ('staged', True, True, True, True)),
    ('f32_split_even', 3): ((512, 1, 'L2', 'L2', 256, 128), ('staged', True, True, True, True)),
    ('f32_split_uneven', 0): ((512, 1, 'L2', 'L2', 224, 128), ('staged', True, True, True, False)),
    ('f32_split_uneven', 3): ((512, 1, 'L2', 'L2', 224, 128), ('staged', True, True, True, False)),
    ('f32_m2', 0): ((512, 2, 'smem', 'smem', 288, 288), ('unstaged', True, 'n/a', False, False)),
    ('f32_m2', 3): ((512, 2, 'smem', 'smem', 288, 288), ('unstaged', True, 'n/a', False, False)),
    ('f32_m2_G_L2', 0): ((512, 2, 'L2', 'smem', 512, 512), ('unstaged', True, False, False, False)),
    ('f32_m2_G_L2', 3): ((512, 2, 'L2', 'smem', 512, 512), ('unstaged', True, False, False, False)),
    ('f64_m0_nondiag', 0): ((512, 0, 'smem', 'smem', 96, 96), ('gemm', True, 'n/a', True, True)),
    ('f64_m0_nondiag', 3): ((512, 0, 'smem', 'smem', 96, 96), ('gemm', True, 'n/a', True, True)),
    ('f64_m0_odd_n', 0): ((512, 0, 'smem', 'smem', 96, 96), ('gemm', True, 'n/a', True, True)),
    ('f64_m0_odd_n', 3): ((512, 0, 'smem', 'smem', 96, 96), ('gemm', True, 'n/a', True, True)),
    ('f64_split_nondiag', 0): ((512, 1, 'L2', 'smem', 160, 80), ('gemm', True, True, True, False)),
    ('f64_split_nondiag', 3): ((512, 1, 'L2', 'smem', 160, 80), ('gemm', True, True, True, False)),
    ('f64_split_odd_n', 0): ((512, 1, 'L2', 'smem', 160, 80), ('gemm', True, True, True, False)),
    ('f64_split_odd_n', 3): ((512, 1, 'L2', 'smem', 160, 80), ('gemm', True, True, True, False)),
    ('f64_m2_nondiag', 0): ((512, 2, 'smem', 'smem', 176, 176), ('gemm', True, 'n/a', False, False)),
    ('f64_m2_nondiag', 3): ((512, 2, 'smem', 'smem', 176, 176), ('gemm', True, 'n/a', False, False)),
    ('f64_m2_odd_n', 0): ((512, 2, 'smem', 'smem', 176, 176), ('gemm', True, 'n/a', False, False)),
    ('f64_m2_odd_n', 3): ((512, 2, 'smem', 'smem', 176, 176), ('gemm', True, 'n/a', False, False)),
}
ELL_PINS = {
    ('m0_staged', 'F_row', 4): (True, True),
    ('m0_staged', 'F_row', 5): (False, True),
    ('m0_staged', 'G_row', 8): (True, True),
    ('m0_staged', 'G_row', 9): (True, False),
    ('m0_staged', 'G_col', 32): (True, True),
    ('m0_staged', 'G_col', 33): (True, False),
    ('m2', 'F_row', 4): (True, True),
    ('m2', 'F_row', 5): (False, True),
    ('m2', 'G_row', 8): (True, True),
    ('m2', 'G_row', 9): (True, False),
    ('m2', 'G_col', 32): (True, True),
    ('m2', 'G_col', 33): (True, False),
}
