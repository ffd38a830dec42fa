"""GPU parity tests: the CUDA path (through the C ABI) vs. the golden vectors
of the unmodified reference and vs. the CPU oracle on seeded inputs.

Tolerances (BASELINE.json north_star): 1e-6 rel fp64, 1e-3 rel fp32 on zhat.

Two kernel families are covered (DESIGN.md section 3): the condensed-KKT kernels
(structured scenes: everything the engine builds) and the dual-form kernels
(dense inputs, and the fp64 backward); `dual_only()` forces the latter.

fp32 (measured, tests/test_oracle.py::test_oracle_matches_reference_on_seeded_baseline_shapes and
scripts/fp32_diag.py): fp32 PDIPM trajectories are chaotic at the 1e-3 level -- after 10 iterations
the iterate is unconverged and the step-length rule is discontinuous. The reference's OWN fp32 result
is within 1e-3 of its fp64 result on 92-96 % of the BASELINE-shape scenes (worst 1.3e-2), and a mere
re-ordering of its BLAS calls (oracle vs reference, both fp32) agrees with it to 1e-3 on 94 % (cfg 3
shapes) to 100 % (cfg 2 shape) of them, worst scene 1.3e-2: on ~2-6 % of the scenes ANY two fp32
implementations land on different trajectories, and they are not the same scenes. A per-scene 1e-3
bound against the fp32 reference is therefore not attainable by any independent implementation;
the gates are, on 48 scenes per shape against outputs of the unmodified reference:
  * at least 95 % of the scenes within 1e-3 + 1.5 |ref32 - ref64| of the fp32 reference (inside the
    tolerance wherever the fp32 reference is itself accurate; at most 2 chaotic outliers in 48),
  * at least 85 % within the plain 1e-3 (the oracle pair: 94-100 %; the reference itself vs fp64: 92-96 %),
  * no scene further than 2e-2 (the oracle pair's worst: 1.3e-2),
  * accuracy against the fp64 reference no worse than the fp32 reference's own: median within 1.2x,
    p90 within 1.2x (+1e-4: the p90 of 48 samples is the 5th largest value).
(The kernel's median error against fp64 is in fact 100x smaller than the reference's.)
"""
import contextlib

import pytest
import torch

from tests.helpers import dual_only, fp32_gate as _fp32_gate, golden_names, load_golden, load_seeded_golden, rel_err, \
    seeded_names

pytestmark = pytest.mark.gpu

GRADS = "dQ dp dG dh dA db dF".split()


def _cuda(ts):
    return tuple(t.cuda() if t is not None else None for t in ts)


PATHS = ["default", "dual"]


def _ctx(path):
    return dual_only() if path == "dual" else contextlib.nullcontext()


# ------------------------------------------------------------------ reference goldens, fp64
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("name", golden_names())
def test_forward_matches_reference_golden_fp64(name, path):
    from lcp_physics_b200 import solve_forward
    inp, ref, max_iter, _ = load_golden(name, torch.float64)
    with _ctx(path):
        zhat, nu, lam, slack, status, iters, resid = solve_forward(*_cuda(inp), max_iter=max_iter)
    assert (status >= 0).all()
    assert rel_err(zhat.cpu(), ref["zhat"]).max() < 1e-6
    # multipliers: loosely pinned (best-iterate choice at the round-off floor, see tests/test_oracle.py)
    assert rel_err(lam.cpu(), ref["lams"]).max() < 5e-3
    assert rel_err(slack.cpu(), ref["slacks"]).max() < 5e-3
    if "nus" in ref:
        assert rel_err(nu.cpu(), ref["nus"]).max() < 5e-3


@pytest.mark.parametrize("name", seeded_names())
def test_forward_matches_reference_seeded_fp64(name):
    """48 scenes at the BASELINE shapes against outputs of the unmodified reference."""
    from lcp_physics_b200 import solve_forward
    inp, ref, max_iter, _ = load_seeded_golden(name)
    zhat = solve_forward(*_cuda(inp), max_iter=max_iter)[0]
    assert rel_err(zhat.cpu(), ref["f64"]["zhat"]).max() < 1e-6


@pytest.mark.parametrize("name", golden_names())
def test_backward_matches_reference_golden_fp64(name):
    """Feed the reference's own saved (zhat, nu, lam, slack) to the CUDA backward (fp64: dual form)."""
    from lcp_physics_b200 import solve_backward
    inp, ref, _, dl = load_golden(name, torch.float64)
    Q, p, G, h, A, b, F = _cuda(inp)
    nu = ref["nus"].cuda() if "nus" in ref else None
    grads = solve_backward(Q, G, A, F, ref["zhat"].cuda(), nu, ref["lams"].cuda(), ref["slacks"].cuda(), dl.cuda())
    # dx (hence dQ, dp, dA, db) is well determined. dlam (hence dG, dh, dF) is the solution of a
    # system whose diagonal s/lam spans 1e+-20 once a scene has converged to the round-off
    # floor: there even a fully pivoted fp64 LU differs from the reference's LAPACK call by 1e-2
    # (measured, DESIGN.md "Parity"); only identical instruction sequences agree. Gate those
    # three on scenes that are not at the floor, and require finiteness everywhere. 1e-4 is the
    # tolerance the oracle itself is pinned at against the reference (tests/test_oracle.py).
    floor = (torch.minimum(ref["slacks"].min(1)[0], ref["lams"].min(1)[0]) < 1e-12)
    for gname, g in zip(GRADS, grads):
        if gname not in ref:
            assert g is None
            continue
        assert torch.isfinite(g).all(), gname
        err = rel_err(g.cpu(), ref[gname])
        if gname in ("dG", "dh", "dF"):
            err = err[~floor]
        if err.numel():
            assert err.max() < 1e-4, (gname, err)


# ------------------------------------------------------------------ reference goldens, fp32
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("name", golden_names())
def test_forward_fp32_golden(name, path):
    """Every small fixture, including the BASELINE shapes (pile_cfg3, pile_cfg3_e3, pile_cfg2_fd3), against the
    fp32 outputs of the unmodified reference, per scene."""
    from lcp_physics_b200 import solve_forward
    inp, ref, max_iter, _ = load_golden(name, torch.float32)
    with _ctx(path):
        zhat = solve_forward(*_cuda(inp), max_iter=max_iter)[0]
    big = name in ("pile_cfg3", "pile_cfg3_e3", "pile_cfg2_fd3")
    # (the dual-form fallback's fp32 LU of the 256 x 256 Schur matrix pivots only inside 32-row blocks: at the
    # BASELINE shapes it is distributionally, not per scene, within 1e-3 -- see test_forward_vs_oracle_seeded_fp32)
    assert rel_err(zhat.cpu(), ref["zhat"]).max() < (1e-2 if (big and path == "dual") else 1e-3)


@pytest.mark.parametrize("name", seeded_names())
def test_forward_fp32_seeded_reference(name):
    """48 scenes at each BASELINE shape against the reference's own fp32 and fp64 outputs."""
    from lcp_physics_b200 import solve_forward
    inp, ref, max_iter, _ = load_seeded_golden(name)
    zhat = solve_forward(*_cuda([t.float() for t in inp]), max_iter=max_iter)[0].cpu()
    _fp32_gate(zhat, ref["f32"]["zhat"], ref["f64"]["zhat"], name)


@pytest.mark.parametrize("name", seeded_names())
def test_backward_fp32_seeded_reference(name):
    """fp32 backward (condensed-KKT kernel) fed with the reference's own fp32 forward state.
    The reference's fp32 gradients are themselves unreliable (measured, DESIGN.md "Parity": against its own fp64
    backward on the same state its dG/dh/dF are off by O(1) on most scenes and dp by up to 1e+1 on single scenes),
    so the truth is the fp64 oracle on that state; the reference's fp32 dp is compared where it is itself sane."""
    from lcp_physics_b200 import solve_backward
    from oracle import pdipm_oracle as po
    inp, ref, _, dl = load_seeded_golden(name)
    r32 = ref["f32"]
    Q, p, G, h, A, b, F = _cuda([t.float() for t in inp])
    e = A.dim() > 1 and A.shape[1] > 0
    nu = r32["nus"].cuda() if "nus" in r32 else None
    grads = solve_backward(Q, G, A if e else None, F, r32["zhat"].cuda(), nu, r32["lams"].cuda(), r32["slacks"].cuda(),
                           dl.float().cuda())
    truth = po.lcp_backward_from_saved(inp, r32["zhat"].double(), r32["nus"].double() if "nus" in r32 else None,
                                       r32["lams"].double(), r32["slacks"].double(), dl)
    for gname, g, t in zip(GRADS, grads, truth):
        if t is None:
            assert g is None
            continue
        assert torch.isfinite(g).all(), gname
        err = rel_err(g.cpu(), t)
        assert err.max() < 1e-3, (gname, err)
        assert err.quantile(0.9) < 1e-4, (gname, err)
    sane = rel_err(r32["dp"], truth[1]) < 1e-4            # where the reference's own fp32 dp agrees with fp64
    assert sane.float().mean() > 0.5
    assert rel_err(grads[1].cpu(), r32["dp"])[sane].max() < 1e-3


# ------------------------------------------------------------------ seeded batches vs the oracle
CONFIGS = {
    # name: (nb, nc, fd, e)   n = 3 nb, m = nc (2 + fd)
    "cfg2_fp64_shape": (16, 32, 3, 0),
    "cfg3_fp32_shape": (32, 64, 2, 0),
    "cfg3_e3": (32, 64, 2, 3),
    "odd_sizes": (5, 7, 2, 3),
}


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_forward_vs_oracle_seeded_fp64(cfg, path):
    from lcp_physics_b200 import solve_forward
    from lcp_physics_b200.scenes import make_scenes
    from oracle import pdipm_oracle as po
    nb, nc, fd, e = CONFIGS[cfg]
    inp = make_scenes(24, nb, nc, fd=fd, e=e, dtype=torch.float64, seed=101)
    ref = po.lcp_forward(*inp, max_iter=10, coupled=False, pivot=False)
    with _ctx(path):
        zhat, nu, lam, slack, status, iters, resid = solve_forward(*_cuda(inp), max_iter=10)
    assert rel_err(zhat.cpu(), ref.zhat).max() < 1e-6
    assert (iters.cpu().long() == ref.info["iters"]).float().mean() > 0.9
    # and against the reference's exact (batch-coupled, pivoted) semantics
    ref2 = po.lcp_forward(*inp, max_iter=10)
    assert rel_err(zhat.cpu(), ref2.zhat).max() < 1e-6


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("cfg", ["cfg2_fp64_shape", "cfg3_fp32_shape", "cfg3_e3"])
def test_forward_vs_oracle_seeded_fp32(cfg, path):
    from lcp_physics_b200 import solve_forward
    from lcp_physics_b200.scenes import make_scenes
    from oracle import pdipm_oracle as po
    nb, nc, fd, e = CONFIGS[cfg]
    inp64 = make_scenes(48, nb, nc, fd=fd, e=e, dtype=torch.float64, seed=202)
    inp32 = tuple(t.float() for t in inp64)
    ref64 = po.lcp_forward(*inp64, max_iter=10).zhat
    ref32 = po.lcp_forward(*inp32, max_iter=10).zhat
    with _ctx(path):
        zhat = solve_forward(*_cuda(inp32), max_iter=10)[0].cpu()
    if path == "default":
        _fp32_gate(zhat, ref32, ref64, cfg)
        return
    # dual-form fallback: fp32 LU of the 256 x 256 Schur matrix with block-local threshold pivoting; its
    # accuracy against fp64 is ~2.6x the LAPACK-pivoted reference's at p90 (DESIGN.md "Parity")
    err, own, mine = rel_err(zhat, ref32), rel_err(ref32, ref64), rel_err(zhat, ref64)
    assert (err < 1e-3).float().mean() >= 0.85, err
    assert float(err.max()) <= 2e-2, err
    assert float(mine.quantile(0.9)) <= max(2e-3, 3 * float(own.quantile(0.9))), (mine, own)


# Block-structure variants of the dual-form look-ahead LU: 2, 3, 6 and 10 diagonal blocks, all-in-shared-memory
# (mode 0), split (mode 1) and the L2-resident plan (mode 2, m = 384 in fp64), with and without equality rows;
# every plan must reproduce the oracle. The same shapes also run through the default (condensed) path.
VARIANTS = {
    # name: (nb, nc, fd, e, dtype, B)
    "m64_fp32_2blocks": (8, 16, 2, 0, torch.float32, 12),
    "m96_fp32_3blocks_e2": (12, 24, 2, 2, torch.float32, 12),
    "m96_fp64_6blocks_e2": (12, 24, 2, 2, torch.float64, 12),
    "m160_fp64_split": (20, 40, 2, 0, torch.float64, 8),
    "m384_fp64_l2_plan": (24, 96, 2, 0, torch.float64, 3),
}


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("name", list(VARIANTS))
def test_plan_variants_match_oracle(name, path):
    from lcp_physics_b200 import solve_forward, _lib
    from lcp_physics_b200.scenes import make_scenes
    from oracle import pdipm_oracle as po
    nb, nc, fd, e, dtype, B = VARIANTS[name]
    inp64 = make_scenes(B, nb, nc, fd=fd, e=e, dtype=torch.float64, seed=77)
    ref = po.lcp_forward(*inp64, max_iter=10).zhat
    inp = tuple(t.to(dtype) for t in inp64)
    n, m = 3 * nb, nc * (2 + fd)
    with _ctx(path):
        zhat = solve_forward(*_cuda(inp), max_iter=10)[0].cpu().double()
        desc = _lib.get_handle(dtype, n, m, e, 0).describe()
    err = rel_err(zhat, ref)
    if dtype == torch.float64:
        assert err.max() < 1e-6, (name, err)
    elif path == "default":
        assert (err < 1e-3).float().mean() >= 0.9 and err.max() < 1e-2, (name, err)     # fp32: see the module docstring
    else:
        assert (err < 1e-3).float().mean() >= 0.8 and err.max() < 2e-2, (name, err)
    if path == "dual":
        assert "condensed KKT: n/a" in desc, desc
        if name == "m384_fp64_l2_plan":
            assert "T:L2" in desc, desc
        if name == "m160_fp64_split":
            assert "split" in desc, desc
    else:
        assert "condensed KKT: N=" in desc, desc


@pytest.mark.parametrize("n,m,e", [(96, 256, 0), (48, 160, 4)])
def test_dense_inputs_at_split_plan_sizes_fp64(n, m, e):
    """Fully dense Q, G, F (no contact structure): the condensed kernel flags every scene as unstructured
    and the dual-form kernel solves them (dense Q inverse, dense Gram GEMMs, dense-GEMV fallbacks of the ELL paths)."""
    from lcp_physics_b200 import solve_forward
    from lcp_physics_b200.scenes import make_dense_random
    from oracle import pdipm_oracle as po
    inp = make_dense_random(3, n, m, e=e, dtype=torch.float64, seed=11)
    ref = po.lcp_forward(*inp, max_iter=10)
    out = solve_forward(*_cuda(inp), max_iter=10)
    assert (out[4] >= 0).all()
    assert rel_err(out[0].cpu(), ref.zhat).max() < 1e-6
    assert bool(torch.isfinite(out[0]).all())


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_mixed_structured_and_dense_scenes_in_one_batch(dtype):
    """The structure test is per scene: engine-structured scenes take the condensed kernel, the others (here: a
    dense F, a dense G row, a non-diagonal Q) fall back to the dual form inside the same call -- forward and backward."""
    from lcp_physics_b200 import solve_forward, solve_backward
    from lcp_physics_b200.scenes import make_scenes
    from oracle import pdipm_oracle as po
    inp = [t.clone() for t in make_scenes(8, 6, 8, fd=2, e=0, dtype=torch.float64, seed=21)]
    Q, p, G, h, A, b, F = inp
    gen = torch.Generator().manual_seed(5)
    W = torch.randn(32, 32, generator=gen, dtype=torch.float64) * 0.05
    F[1] += W @ W.t()                                  # dense PSD F
    G[3, 0, :] = torch.randn(18, generator=gen, dtype=torch.float64) * 0.1   # one dense row of G (> 8 non-zeros)
    Q[5, 0, 1] = Q[5, 1, 0] = 0.05                     # non-diagonal (still SPD) Q
    ref = po.lcp_forward(*inp, max_iter=10, coupled=False)
    dev = _cuda([t.to(dtype) for t in inp])
    zhat, nu, lam, slack, status, iters, resid = solve_forward(*dev, max_iter=10)
    assert (status >= 0).all()
    err = rel_err(zhat.cpu(), ref.zhat)
    if dtype == torch.float64:
        assert err.max() < 1e-6
    else:
        unstructured = torch.tensor([False, True, False, True, False, True, False, False])
        assert err[~unstructured].max() < 1e-3          # condensed kernel
        assert err[unstructured].max() < 1e-2           # dual-form fp32 fallback (block-local pivoting)
    g = torch.randn(8, 18, generator=gen, dtype=torch.float64)
    grads = solve_backward(dev[0], dev[2], None, dev[6], zhat, None, lam, slack, g.to(dtype).cuda())
    truth = po.lcp_backward_from_saved(inp, zhat.double().cpu(), None, lam.double().cpu(), slack.double().cpu(), g)
    # scenes converged to the round-off floor (lambda, s ~ 1e-16 in fp64): d = lambda/s is noise there and so are
    # the gradients of ANY implementation (the reference's included); finiteness is required everywhere (this
    # also exercises the rescue pass: the dual LU breaks down on one of these scenes)
    floor = (torch.minimum(slack.min(1)[0], lam.min(1)[0]) < 1e-12).cpu()
    for gname, a, t in zip(GRADS, grads, truth):
        if t is None:
            continue
        assert torch.isfinite(a).all(), gname
        if gname in ("dQ", "dp") and bool((~floor).any()):
            assert rel_err(a.cpu(), t)[~floor].max() < (1e-4 if dtype == torch.float64 else 5e-3), gname


def test_poststabilisation_and_fd3_block_shapes_fp64():
    """Component sizes 1 (post-stabilisation: F = 0) and 5 (three friction directions) of the condensed kernel."""
    from lcp_physics_b200 import solve_forward, _lib
    from oracle import pdipm_oracle as po
    inp, ref, max_iter, _ = load_golden("poststab", torch.float64)
    out = solve_forward(*_cuda(inp), max_iter=max_iter)
    assert rel_err(out[0].cpu(), ref["zhat"]).max() < 1e-6
    assert "condensed KKT: N=" in _lib.get_handle(torch.float64, inp[0].shape[1], inp[2].shape[1], inp[4].shape[1], 0).describe()
    inp, ref, max_iter, _ = load_golden("pile_cfg2_fd3", torch.float64)
    out = solve_forward(*_cuda(inp), max_iter=max_iter)
    assert rel_err(out[0].cpu(), po.lcp_forward(*inp, max_iter=max_iter).zhat).max() < 1e-6


# ------------------------------------------------------------------ autograd, host path, invariants
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_autograd_through_lcpfunction_matches_oracle(dtype):
    from lcp_physics_b200 import LCPFunction
    from lcp_physics_b200.scenes import make_scenes
    from oracle import pdipm_oracle as po
    inp = make_scenes(6, 6, 7, fd=2, e=3, dtype=torch.float64, seed=5)
    leaves = [t.to(dtype).cuda().requires_grad_(True) for t in inp]
    fn = LCPFunction(max_iter=6)
    zhat = fn(*leaves)
    g = torch.randn(zhat.shape, dtype=torch.float64, generator=torch.Generator().manual_seed(1))
    (zhat * g.to(dtype).cuda()).sum().backward()
    ref = po.lcp_forward(*inp, max_iter=6, coupled=False, pivot=False)
    rg = po.lcp_backward_from_saved(inp, zhat.detach().double().cpu(), fn.nus.double().cpu(), fn.lams.double().cpu(),
                                    fn.slacks.double().cpu(), g, pivot=False)
    ftol, gtol = (1e-6, 1e-4) if dtype == torch.float64 else (1e-3, 1e-3)
    assert rel_err(zhat.detach().cpu(), ref.zhat).max() < ftol
    for leaf, r, nm in zip(leaves, rg, GRADS):
        assert leaf.grad is not None, nm
        assert rel_err(leaf.grad.cpu(), r).max() < gtol, nm


@pytest.mark.parametrize("e", [0, 3])
def test_exact_adjoint_matches_finite_differences_fp64(e):
    """LCPB200_BWD_EXACT_ADJOINT (SURVEY.md f-4): gradients of l = g . zhat against central finite differences of
    the converged forward solve, along random directions of p, F (on its non-zero pattern) and of the
    contact-normal rows of h and G (the +-tangent friction rows are linearly dependent, J_f2 = -J_f1: the solution
    map is not differentiable w.r.t. independent perturbations of those rows). The reference's (bug-compatible)
    gradients fail the same check when F != 0 (SURVEY.md F6)."""
    from lcp_physics_b200 import solve_forward, solve_backward
    from lcp_physics_b200.scenes import make_scenes
    from oracle import pdipm_oracle as po
    nc = 6
    inp = make_scenes(5, 5, nc, fd=2, e=e, dtype=torch.float64, seed=33)
    Q, p, G, h, A, b, F = inp
    gen = torch.Generator().manual_seed(7)
    g = torch.randn(5, 15, generator=gen, dtype=torch.float64)
    kw = dict(max_iter=40, eps=1e-10)

    def loss(args):
        z = solve_forward(*_cuda(args), **kw)[0].cpu()
        return (z * g).sum(1)

    out = solve_forward(*_cuda(inp), **kw)
    assert (out[6] < 1e-8).all()                                  # converged (best residual)
    dev = _cuda(inp)
    nu = out[1] if e > 0 else None
    exact = solve_backward(dev[0], dev[2], dev[4] if e else None, dev[6], out[0], nu, out[2], out[3], g.cuda(),
                           exact_adjoint=True)
    compat = solve_backward(dev[0], dev[2], dev[4] if e else None, dev[6], out[0], nu, out[2], out[3], g.cuda())
    ora = po.lcp_backward_exact_from_saved(inp, out[0].cpu(), nu.cpu() if e else None, out[2].cpu(), out[3].cpu(), g)
    eps = 1e-5
    worst_exact, worst_compat = 0.0, 0.0
    for k, name in ((1, "dp"), (3, "dh"), (2, "dG"), (6, "dF")):
        d = torch.randn(inp[k].shape, generator=gen, dtype=torch.float64) * (inp[k] != 0 if k in (2, 6) else 1.0)
        if k in (2, 3):
            d[:, nc:] = 0                                        # contact-normal rows only
        plus = [t.clone() for t in inp]; minus = [t.clone() for t in inp]
        plus[k] += eps * d; minus[k] -= eps * d
        fd = (loss(plus) - loss(minus)) / (2 * eps)
        an_exact = (exact[k].cpu() * d).flatten(1).sum(1)
        an_compat = (compat[k].cpu() * d).flatten(1).sum(1)
        scale = fd.abs().max()
        worst_exact = max(worst_exact, float((an_exact - fd).abs().max() / scale))
        worst_compat = max(worst_compat, float((an_compat - fd).abs().max() / scale))
        # CUDA vs the oracle's restatement of the same (transposed) system; the state is converged, so
        # d = lambda/s spans 1e+-10 and dlam (dh, dG, dF) carries the KKT conditioning noise of tests/test_oracle.py
        assert rel_err(exact[k].cpu(), ora[k]).max() < (1e-6 if name == "dp" else 2e-3), name
    assert worst_exact < 2e-3, worst_exact
    assert worst_compat > 5 * worst_exact, (worst_compat, worst_exact)


def test_host_buffers_equal_device_buffers():
    """CPU tensors go through lcpb200_forward_host / backward_host (chunked copy+solve pipeline), including the
    retained-state backward (Q == NULL) that bench.py's e2e leg uses."""
    from lcp_physics_b200 import solve_forward, solve_backward
    from lcp_physics_b200.scenes import make_scenes
    inp = make_scenes(700, 4, 4, fd=2, e=3, dtype=torch.float32, seed=9)
    saved = {}
    out_h = solve_forward(*inp, max_iter=10, save=saved)
    out_d = solve_forward(*_cuda(inp), max_iter=10)
    for a, b in zip(out_h, out_d):
        assert a.device.type == "cpu"
        assert torch.equal(a, b.cpu())
    assert torch.isfinite(out_h[0]).all()
    Q, p, G, h, A, b, F = inp
    g = torch.randn(700, 12)
    gr = solve_backward(Q, G, A, F, out_h[0], out_h[1], out_h[2], out_h[3], g, saved=saved)   # retained device state
    gh = solve_backward(Q, G, A, F, out_h[0], out_h[1], out_h[2], out_h[3], g)                # full upload
    gd = solve_backward(*_cuda((Q, G, A, F, out_h[0], out_h[1], out_h[2], out_h[3], g)))
    for a, b, c in zip(gh, gd, gr):
        assert torch.allclose(a, b.cpu(), rtol=0, atol=0, equal_nan=True)
        assert torch.allclose(c, b.cpu(), rtol=0, atol=0, equal_nan=True)


def test_batch_of_one_equals_batch_of_many():
    """Scenes are independent: solving a scene alone or inside a batch is bit-identical (both kernel families)."""
    from lcp_physics_b200 import solve_forward
    from lcp_physics_b200.scenes import make_scenes
    for path in PATHS:
        with _ctx(path):
            inp = _cuda(make_scenes(5, 8, 12, fd=2, e=0, dtype=torch.float64, seed=3))
            full = solve_forward(*inp, max_iter=10)[0]
            for k in range(5):
                one = solve_forward(*[t[k:k + 1] if t.dim() > 1 else t for t in inp], max_iter=10)[0]
                assert torch.equal(one[0], full[k])


def test_repeated_calls_are_bitwise_reproducible_fp32():
    from lcp_physics_b200 import solve_forward, solve_backward
    from lcp_physics_b200.scenes import make_scenes
    inp = _cuda(make_scenes(600, 32, 64, fd=2, e=0, dtype=torch.float32, seed=4))
    g = torch.randn(600, 96, device="cuda")
    a = solve_forward(*inp, max_iter=10)
    ga = solve_backward(inp[0], inp[2], None, inp[6], a[0], None, a[2], a[3], g)
    b = solve_forward(*inp, max_iter=10)
    gb = solve_backward(inp[0], inp[2], None, inp[6], b[0], None, b[2], b[3], g)
    assert torch.equal(a[0], b[0]) and torch.equal(a[2], b[2])
    for x, y in zip(ga, gb):
        if x is not None:
            assert torch.equal(x, y)


def test_singular_q_raises_reference_error():
    from lcp_physics_b200 import LCPFunction
    from lcp_physics_b200.scenes import make_scenes
    inp = list(_cuda(make_scenes(3, 4, 4, fd=2, e=0, dtype=torch.float64, seed=3)))
    inp[0] = inp[0].clone()
    inp[0][1] = 0
    with pytest.raises(RuntimeError, match="Cannot perform LU factorization on Q"):
        LCPFunction()(*inp)


def test_empty_batch_and_zero_iterations():
    from lcp_physics_b200 import solve_forward
    from lcp_physics_b200.scenes import make_scenes
    inp = _cuda(make_scenes(2, 4, 4, fd=2, e=0, dtype=torch.float64, seed=3))
    empty = tuple(t[:0] if t.dim() > 1 else t for t in inp)
    out = solve_forward(*empty)
    assert out[0].shape == (0, 12)
    out0 = solve_forward(*inp, max_iter=0)
    assert (out0[5] == 0).all()


def test_residual_property_full_size_cfg3():
    """Size-independent property at the BASELINE size (B=4096 x 64 contacts, fp32):
    the returned (zhat, lam, slack) satisfies the LCP residual it reports."""
    from lcp_physics_b200 import solve_forward
    from lcp_physics_b200.scenes import make_scenes
    B = 4096
    inp = _cuda(make_scenes(B, 32, 64, fd=2, e=0, dtype=torch.float32, seed=7))
    Q, p, G, h, A, b, F = inp
    zhat, nu, lam, slack, status, iters, resid = solve_forward(*inp, max_iter=10)
    assert torch.isfinite(zhat).all()
    assert (status >= 0).all()
    assert (lam > 0).all() and (slack > 0).all()
    rx = torch.bmm(G.transpose(1, 2), lam.unsqueeze(2)).squeeze(2) + torch.bmm(Q, zhat.unsqueeze(2)).squeeze(2) + p
    rz = torch.bmm(G, zhat.unsqueeze(2)).squeeze(2) + slack - h - torch.bmm(F, lam.unsqueeze(2)).squeeze(2)
    mu = (lam * slack).sum(1).abs() / lam.shape[1]
    r = rx.norm(dim=1) + rz.norm(dim=1) + lam.shape[1] * mu
    assert torch.allclose(r, resid, rtol=5e-2, atol=1e-4)
    assert (iters > 0).all() and (iters <= 10).all()


def test_full_size_cfg2_fp64_sample_matches_oracle():
    """BASELINE config 2 (forward only, B=1024, 32 contacts x 3 friction directions, fp64): a 32-scene sample of
    the full batch against the oracle at 1e-6."""
    from lcp_physics_b200 import solve_forward
    from lcp_physics_b200.scenes import make_scenes
    from oracle import pdipm_oracle as po
    inp = make_scenes(1024, 16, 32, fd=3, e=0, dtype=torch.float64, seed=8)
    out = solve_forward(*_cuda(inp), max_iter=10)
    assert (out[4] >= 0).all() and torch.isfinite(out[0]).all()
    idx = torch.arange(0, 1024, 32)
    sub = tuple(t[idx] if t.dim() > 1 else t for t in inp)
    ref = po.lcp_forward(*sub, max_iter=10, coupled=False)
    assert rel_err(out[0].cpu()[idx], ref.zhat).max() < 1e-6


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_backward_with_reused_structure_is_bitwise_the_same(dtype):
    """LCPB200_BWD_REUSE_STRUCTURE: the backward that reads the block structure its forward saved (19 KB per scene
    at cfg 3) returns bit-for-bit the gradients of the backward that scans Q, G, F again -- also when some scenes of
    the batch have no structure (dense F / dense G row / non-diagonal Q: left to the dual form) and when another
    forward on the same handle invalidates the token (falls back to scanning)."""
    from lcp_physics_b200 import solve_forward, solve_backward
    from lcp_physics_b200.scenes import make_scenes
    inp = [t.clone() for t in make_scenes(24, 32, 64, fd=2, e=0, dtype=torch.float64, seed=31)]
    Q, p, G, h, A, b, F = inp
    gen = torch.Generator().manual_seed(7)
    W = torch.randn(256, 256, generator=gen, dtype=torch.float64) * 0.02
    F[2] += W @ W.t()
    Q[9, 0, 1] = Q[9, 1, 0] = 0.05
    dev = _cuda([t.to(dtype) for t in inp])
    g = torch.randn(24, 96, generator=gen, dtype=torch.float64).to(dtype).cuda()
    saved = {}
    out = solve_forward(*dev, max_iter=10, save=saved)
    assert "struct" in saved
    reused = solve_backward(dev[0], dev[2], None, dev[6], out[0], None, out[2], out[3], g, saved=saved)
    scanned = solve_backward(dev[0], dev[2], None, dev[6], out[0], None, out[2], out[3], g)
    for name, a, c in zip(GRADS, reused, scanned):
        if a is not None:
            assert torch.equal(a, c), name
    # a second forward (other inputs, same shapes) on the handle: the old token must not be honoured
    other = _cuda([t.to(dtype) for t in make_scenes(24, 32, 64, fd=2, e=0, dtype=torch.float64, seed=32)])
    solve_forward(*other, max_iter=10, save={})
    stale = solve_backward(dev[0], dev[2], None, dev[6], out[0], None, out[2], out[3], g, saved=saved)
    for name, a, c in zip(GRADS, stale, scanned):
        if a is not None:
            assert torch.equal(a, c), name
