"""GPU: the dual-form kernels (DESIGN.md section 3.3) at every plan tier, per-scene branch, sparse-copy limit and
backward path, and with several scenes per CTA.

Every test runs under `dual_only()` unless it says otherwise, and first proves which plan ran: the dual-form part
of `Handle.describe()` equals the host restatement's (tests/dual_plan.py; tests/test_dual_plan.py pins the tiers and
per-scene verdicts of every shape used here).

* every tier (threads 128 / 256 / 512, T in shared memory, split evenly, split unevenly or padded, in L2; G and
  Q^-1 in each residency) and every R-forming branch (staged Gram, unstaged Gram, general GEMM for a non-diagonal Q
  or n % VC != 0), with and without equality rows: fp64 forward against the oracle, both adjoints on the kernel's
  own state; fp32 per scene after one iteration, distributionally after 10, and the fp32 backward on its own state;
* the ELL limits on both sides: 4 / 5 non-zeros in an F row, 8 / 9 in a G row, 32 / 33 in a G column;
* several scenes per CTA (B = 2 grid + 3): every scene bitwise equal to the same scene solved alone, forward and
  both adjoints, with singular-Q, non-finite, dense-F, dense-G and non-diagonal-Q scenes among them;
* the host pipeline's retained state (the saved R) against the full upload and the device path, both adjoints and a
  subset of the gradients; LCPB200_DUAL_BACKWARD on a shape with a condensed plan; workspace growth on one handle.
"""
import os

import pytest
import torch

from tests import dual_plan as dp
from tests.helpers import dual_only, rel_err

pytestmark = pytest.mark.gpu
GRADS = "dQ dp dG dh dA db dF".split()


def _handle(dtype, n, m, e, host=False):
    from lcp_physics_b200 import _lib
    return _lib.get_handle(dtype, n, m, e, torch.cuda.current_device(),
                           "host" if host else torch.cuda.current_stream().cuda_stream)


def _check_plan(dtype, inp, host=False):
    """The handle's dual-form plan is the restatement's; returns (plan, grid)."""
    n, m, e = dp.sizes(inp)
    plan = dp.make_plan(4 if dtype == torch.float32 else 8, n, m, e)
    desc = _handle(dtype, n, m, e, host).describe()
    assert dp.describe(plan) in desc, (dp.describe(plan), desc)
    print("describe:", desc)
    return plan, int(desc.split("grid<=")[-1].split()[0])


def _oracle(inp, max_iter=10):
    from oracle import pdipm_oracle as po
    return po.lcp_forward(*inp, max_iter=max_iter, coupled=False, pivot=False)


def _forward(inp, dtype, max_iter=10, **kw):
    from lcp_physics_b200 import solve_forward
    out = solve_forward(*[t.to(dtype).cuda() for t in inp], max_iter=max_iter, **kw)
    torch.cuda.synchronize()
    return out


def _backward(inp, dtype, state, g, exact, **kw):
    from lcp_physics_b200 import solve_backward
    Q, p, G, h, A, b, F = [t.to(dtype).cuda() for t in inp]
    e = dp.sizes(inp)[2]
    zhat, nu, lam, slack = state
    out = solve_backward(Q, G, A if e else None, F, zhat, nu, lam, slack, g.to(dtype).cuda(), exact_adjoint=exact, **kw)
    torch.cuda.synchronize()
    return out


def _gz(B, n, seed=3):
    return torch.randn(B, n, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


def _grad_errors(inp, dtype, state, g):
    """Both adjoints on `state` (the kernel's own) against the oracle's: {(exact, name): per-scene rel err}."""
    from oracle import pdipm_oracle as po
    s64 = [t.double().cpu() if t is not None else None for t in state]
    out = {}
    for exact, ora in ((False, po.lcp_backward_from_saved), (True, po.lcp_backward_exact_from_saved)):
        got = _backward(inp, dtype, state, g, exact)
        truth = ora(inp, *s64, g)
        for name, a, t in zip(GRADS, got, truth):
            if t is None:
                assert a is None
                continue
            assert torch.isfinite(a).all(), (name, exact)
            out[(exact, name)] = rel_err(a.cpu(), t)
    return out


def check_fp64(inp):
    out = _forward(inp, torch.float64)
    assert (out[4] >= 0).all()
    fwd = float(rel_err(out[0].cpu(), _oracle(inp).zhat).max())
    assert fwd < 1e-6, fwd
    state = _forward(inp, torch.float64, max_iter=5)[:4]
    errs = _grad_errors(inp, torch.float64, state, _gz(inp[0].shape[0], inp[0].shape[1]))
    worst = max(float(v.max()) for v in errs.values())
    print("fp64 forward %.2e gradients %.2e" % (fwd, worst))
    assert worst < 1e-6, {k: float(v.max()) for k, v in errs.items()}


def check_fp32(inp):
    B = inp[0].shape[0]
    one, ref1 = _forward(inp, torch.float32, max_iter=1), _oracle(inp, max_iter=1)
    for k, name in ((0, "zhat"), (2, "lams"), (3, "slacks")):
        err = rel_err(one[k].cpu(), getattr(ref1, name))
        assert err.max() < 1e-4, (name, err)
    zhat = _forward(inp, torch.float32)[0].cpu()
    ref64, ref32 = _oracle(inp).zhat, _oracle([t.float() for t in inp]).zhat
    err, own, mine = rel_err(zhat, ref32), rel_err(ref32, ref64), rel_err(zhat, ref64)
    assert (err < 1e-3).float().mean() >= 0.85, err             # test_forward_vs_oracle_seeded_fp32[*-dual]
    assert float(err.max()) <= 2e-2, err
    # a median, not test_forward_vs_oracle_seeded_fp32's p90: of 8 scenes one chaotic scene is the p90
    assert float(mine.median()) <= max(1e-3, 3 * float(own.median())), (mine, own)
    state = _forward(inp, torch.float32, max_iter=5)[:4]
    errs = _grad_errors(inp, torch.float32, state, _gz(B, inp[0].shape[1]))
    print("fp32 forward %.2e gradients max %.2e" % (float(mine.max()), max(float(v.max()) for v in errs.values())))
    for k, v in errs.items():
        assert v.max() < 1e-3 and v.median() < 1e-4, (k, v)        # max as test_backward_fp32_seeded_reference


# ------------------------------------------------------------------ every tier and every prefactor branch
# name: (dtype, nb, nc, variant) with engine scenes of fd = 2 (n = 3 nb, m = 4 nc); variant "diag" (the engine's
# diagonal Q) or "nondiag" (dp.nondiag_q); an odd nb gives n % VC != 0 in fp64
TIERS = {
    "f64_m0_nt128": (torch.float64, 8, 8, "diag"),
    "f64_m0_nt256": (torch.float64, 16, 14, "diag"),
    "f64_m0_nt512": (torch.float64, 16, 24, "diag"),
    "f64_m0_unstaged": (torch.float64, 32, 10, "diag"),
    "f64_m0_G_L2": (torch.float64, 16, 34, "diag"),
    "f64_m0_G_L2_Qi_L2": (torch.float64, 24, 33, "diag"),
    "f64_split_even": (torch.float64, 20, 40, "diag"),
    "f64_split_padded": (torch.float64, 16, 37, "diag"),
    "f64_m2": (torch.float64, 16, 44, "diag"),
    "f64_m2_Qi_L2": (torch.float64, 32, 50, "diag"),
    "f64_m2_G_L2": (torch.float64, 40, 50, "diag"),
    "f64_m2_G_L2_Qi_L2": (torch.float64, 50, 60, "diag"),
    "f32_m0_nt128": (torch.float32, 8, 8, "diag"),
    "f32_m0_nt256": (torch.float32, 16, 12, "diag"),
    "f32_m0_nt512": (torch.float32, 16, 24, "diag"),
    "f32_m0_G_L2": (torch.float32, 32, 42, "diag"),
    "f32_split_even": (torch.float32, 32, 64, "diag"),
    "f32_split_uneven": (torch.float32, 32, 50, "diag"),
    "f32_m2": (torch.float32, 32, 70, "diag"),
    "f32_m2_G_L2": (torch.float32, 32, 124, "diag"),
}
# the R-forming branches at a mode-0, a split and an L2 shape (fp64)
for _name, _nc in (("m0", 24), ("split", 37), ("m2", 44)):
    TIERS["f64_%s_nondiag" % _name] = (torch.float64, 16, _nc, "nondiag")
    TIERS["f64_%s_odd_n" % _name] = (torch.float64, 15, _nc, "diag")


def build_tier(name, e, B):
    dtype, nb, nc, variant = TIERS[name]
    inp = dp.engine_scenes(B, nb, nc, 2, e=e, seed=300 + nb + nc)
    return dtype, (dp.nondiag_q(inp) if variant == "nondiag" else inp)


@pytest.mark.parametrize("e", [0, 3])
@pytest.mark.parametrize("name", list(TIERS))
def test_tier_against_oracle(name, e):
    dtype, inp = build_tier(name, e, 2 if TIERS[name][0] == torch.float64 else 8)
    with dual_only():
        _check_plan(dtype, inp)
        (check_fp64 if dtype == torch.float64 else check_fp32)(inp)


# ------------------------------------------------------------------ ELL limits
# G in L2 at a staged mode-0 shape (the G copies are built from the staged G) and at a mode-2 shape (from global G)
ELL_SHAPES = {"m0_staged": (16, 34), "m2": (40, 50)}


def build_ell(shape, which, k, B=2):
    nb, nc = ELL_SHAPES[shape]
    inp = dp.engine_scenes(B, nb, nc, 2, seed=400 + nb)
    m = 4 * nc
    if which == "F_row":
        return dp.f_row_nnz(inp, m - 1, k)              # a gamma row: mu and two friction entries
    if which == "G_row":
        return dp.g_row_nnz(inp, nc, k)                 # a friction row: six entries
    return dp.g_col_nnz(inp, 1, k)                      # body 0's x column


ELL_CASES = [("F_row", 4), ("F_row", 5), ("G_row", 8), ("G_row", 9), ("G_col", 32), ("G_col", 33)]


@pytest.mark.parametrize("which,k", ELL_CASES)
@pytest.mark.parametrize("shape", list(ELL_SHAPES))
def test_ell_limits(shape, which, k):
    inp = build_ell(shape, which, k)
    with dual_only():
        _check_plan(torch.float64, inp)
        check_fp64(inp)


# ------------------------------------------------------------------ several scenes per CTA
MULTI_SHAPES = {   # (dtype, nb, nc): mp != m everywhere, so that the padded tails of the vectors are in play
    "f64_m0": (torch.float64, 16, 34), "f64_split": (torch.float64, 16, 37), "f64_m2": (torch.float64, 40, 50),
    "f32_m0": (torch.float32, 32, 42), "f32_split": (torch.float32, 32, 50), "f32_m2": (torch.float32, 32, 70),
}


def multi_kinds(nb, nc):
    """The distinct scenes of the multi-scene batch, one per kind (each a batch of one)."""
    base = dp.engine_scenes(6, nb, nc, 2, seed=500 + nb)
    one = lambda inp, s: tuple(t[s:s + 1] if t.dim() > 1 else t for t in inp)
    m = 4 * nc
    return {
        "singular_q": one(dp.singular_q(base, [0]), 0),
        "nonfinite_h": one(dp.nonfinite_h(base, [1]), 1),
        "diag": one(base, 2),
        "nondiag_q": one(dp.nondiag_q(base), 3),
        "dense_F": one(dp.f_row_nnz(base, m - 1, 5), 4),
        "dense_G": one(dp.g_col_nnz(base, 1, 33), 5),
    }


def multi_order(grid, K):
    """Kind of every scene of a batch of 2 grid + 3: CTA c meets kinds (c % K, (c // K) % K, ...) in turn, so every
    ordered pair of kinds follows each other on some CTA (K^2 <= grid)."""
    assert K * K <= grid
    B = 2 * grid + 3
    return [(s % grid) % K if s < grid else ((s % grid) // K + (s // grid) - 1) % K for s in range(B)]


def _bits(t):
    if t is None:
        return None
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int64) if t.is_floating_point() else t


def _same(a, b):
    return (a is None and b is None) or torch.equal(_bits(a), _bits(b))


@pytest.mark.parametrize("shape", list(MULTI_SHAPES))
def test_several_scenes_per_cta_bitwise(shape):
    dtype, nb, nc = MULTI_SHAPES[shape]
    kinds = multi_kinds(nb, nc)
    names = list(kinds)
    with dual_only():
        _, grid = _check_plan(dtype, kinds["diag"])
        order = multi_order(grid, len(names))
        batch = dp.cat(*[kinds[names[k]] for k in order])
        full = _forward(batch, dtype)
        st = full[4].cpu()
        assert all(int(st[s]) == -1 for s, k in enumerate(order) if names[k] == "singular_q")
        g = _gz(len(names), 3 * nb)[order]             # every occurrence of a kind: the same state and g
        gfull = {ex: _backward(batch, dtype, full[:4], g, ex) for ex in (False, True)}
        for k, name in enumerate(names):
            idx = [s for s, kk in enumerate(order) if kk == k]
            alone = _forward(kinds[name], dtype)
            for a, b in zip(full, alone):
                for s in idx:
                    assert _same(None if a is None else a[s:s + 1], b), (shape, name, s)
            st1 = [None if t is None else t[idx[:1]] for t in full[:4]]
            for ex in (False, True):
                g1 = _backward(kinds[name], dtype, st1, g[idx[:1]], ex)
                for gname, a, b in zip(GRADS, gfull[ex], g1):
                    for s in idx:
                        assert _same(None if a is None else a[s:s + 1], b), (shape, name, gname, ex, s)


# ------------------------------------------------------------------ host pipeline with the saved R
HOST_CASES = {   # name: (nb, nc, e, dual_only): a split shape, and n + e > 128 (no condensed plan at all)
    "split_e3": (16, 37, 3, True),
    "n150_e3": (50, 30, 3, False),
}


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("name", list(HOST_CASES))
def test_host_pipeline_saved_r(name, dtype):
    """forward_host keeps R when no condensed plan exists; backward_host on the retained state then reuses it -- but
    not under the exact adjoint, whose R holds F^T."""
    import contextlib
    from lcp_physics_b200 import solve_backward, solve_forward
    nb, nc, e, force = HOST_CASES[name]
    B = 6
    inp = [t.to(dtype) for t in dp.engine_scenes(B, nb, nc, 2, e=e, seed=600 + nb)]
    with dual_only() if force else contextlib.nullcontext():
        plan, _ = _check_plan(dtype, inp, host=True)
        assert "condensed KKT: n/a" in _handle(dtype, *dp.sizes(inp), host=True).describe()
        Q, p, G, h, A, b, F = inp
        g = _gz(B, 3 * nb).to(dtype)
        res = {}
        for exact in (False, True):
            saved = {}
            out = solve_forward(*inp, max_iter=5, save=saved)
            assert out[0].device.type == "cpu" and (out[4] >= 0).all()
            st = out[:4]
            retained = solve_backward(Q, G, A, F, *st, g, saved=saved, exact_adjoint=exact)
            upload = solve_backward(Q, G, A, F, *st, g, exact_adjoint=exact)
            device = solve_backward(*[t.cuda() for t in (Q, G, A, F, *st, g)], exact_adjoint=exact)
            for gname, r, u, d in zip(GRADS, retained, upload, device):
                assert _same(r, u) and _same(r, None if d is None else d.cpu()), (gname, exact)
            res[exact] = retained
            # a subset of the gradients: the rest are not computed
            saved = {}
            solve_forward(*inp, max_iter=5, save=saved)
            need = (False, True, False, True, False, True, False)
            part = solve_backward(Q, G, A, F, *st, g, need=need, saved=saved, exact_adjoint=exact)
            for gname, want, a, full in zip(GRADS, need, part, retained):
                assert (a is None) if not want else _same(a, full), (gname, exact)
        # F != 0: the exact adjoint is not the reference's gradient (the saved R, which holds F, was not reused)
        assert not torch.equal(res[False][1], res[True][1])
        assert float(rel_err(res[False][1], res[True][1]).min()) > 1e-6


# ------------------------------------------------------------------ LCPB200_DUAL_BACKWARD, workspace growth
def test_dual_backward_switch_fp32():
    """On a shape with a condensed plan, LCPB200_DUAL_BACKWARD=1 routes the fp32 backward to the dual form; both
    backwards meet the fp32 backward gates against the fp64 oracle on the same fp32 state."""
    from oracle import pdipm_oracle as po
    inp = dp.engine_scenes(8, 16, 24, 2, e=3, seed=700)
    n, m, e = dp.sizes(inp)
    assert "condensed KKT: N=" in _handle(torch.float32, n, m, e).describe()
    state = _forward(inp, torch.float32, max_iter=5)[:4]
    g = _gz(8, n)
    truth = po.lcp_backward_from_saved(inp, *[t.double().cpu() for t in state], g)
    cond = _backward(inp, torch.float32, state, g, False)
    assert cond[1] is not None
    os.environ["LCPB200_DUAL_BACKWARD"] = "1"
    try:
        dual = _backward(inp, torch.float32, state, g, False)
    finally:
        del os.environ["LCPB200_DUAL_BACKWARD"]
    for name, a, c, t in zip(GRADS, cond, dual, truth):
        if t is None:
            continue
        for x in (a, c):
            err = rel_err(x.cpu(), t)
            assert err.max() < 1e-3 and err.quantile(0.9) < 1e-4, (name, err)


def test_workspace_growth_on_one_handle():
    """B = 1, then B = grid + 5 (the workspace grows to every resident CTA), then B = 1 on one handle: bitwise the
    results of fresh handles."""
    from lcp_physics_b200 import _lib
    with dual_only():
        one = dp.engine_scenes(1, 16, 34, 2, seed=800)
        _, grid = _check_plan(torch.float64, one)
        many = dp.engine_scenes(grid + 5, 16, 34, 2, seed=801)
        got = [_forward(x, torch.float64) for x in (one, many, one)]
        for x, out in zip((one, many, one), got):
            _lib.clear_handles()
            ref = _forward(x, torch.float64)
            for a, b in zip(out, ref):
                assert _same(a, b)
