"""GPU: exact-adjoint gradients (the transposed KKT system, DESIGN.md section 3.4) through the engine path, the large-
scene kernel, `BatchedWorld` and `B200PdipmEngine`.

* the fused engine backward (condensed kernel) against an independent implementation: the dense assembly
  (`assemble_contacts`, autograd through its adjoint kernel) + `LCPFunction(exact_adjoint=True)`;
* the banded kernel against the condensed kernel, both exact; in post-stabilisation (F = 0) the banded exact and
  bug-compatible gradients are bitwise equal;
* central finite differences of one converged engine solve, on the condensed and on the banded kernel: the exact
  gradients match, the reference's (bug-compatible) ones are worse along the friction coefficients;
* central differences of 6-step `BatchedWorld(exact_adjoint=True)` rollouts whose solves all converge (sliding
  contacts), on both kernels, and the fp32 rollout against fp64; the flag never changes a trajectory;
* `B200PdipmEngine(exact_adjoint=True)` fused against dense on recorded reference worlds, and a replaced
  `lcp_solver` refuses the flag.
"""
import os

import numpy as np
import pytest
import torch

from tests.helpers import ReplayWorld, load_world_records, rel_err

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bworld_large.npz")
NAMES = ["mass", "inertia", "v", "fext", "normal", "p1", "p2", "mu", "restitution"]
DT = 1.0 / 30


@pytest.fixture
def forced_banded():
    from lcp_physics_b200 import _lib

    def set_(on):
        if on:
            os.environ["LCPB200_FORCE_BANDED"] = "1"
        else:
            os.environ.pop("LCPB200_FORCE_BANDED", None)
        _lib.clear_handles()
    yield set_
    set_(False)


def _soa_scene(B, nb, nc, seed):
    from lcp_physics_b200.scenes import make_contact_soa
    soa = dict(make_contact_soa(B, nb, nc, seed=seed))
    fext = torch.zeros(B, 3 * nb, dtype=torch.float64)
    fext[:, 2::3] = 10.0 * soa["mass"]
    soa["fext"] = fext
    return soa


def _pins(B, e, n):
    A = torch.zeros(B, e, n, dtype=torch.float64)
    A[:, torch.arange(e), torch.arange(e)] = 1
    return A.cuda(), torch.zeros(B, e, dtype=torch.float64).cuda()


def _grads(leaves):
    return [t.grad.detach().cpu() if t.grad is not None else torch.zeros(t.shape, dtype=t.dtype) for t in leaves]


# ------------------------------------------------------------------ 1. fused engine vs dense path (condensed)
def _fused_grads(soa, b1, b2, A0, b0, mode, exact, gz, max_iter=5, counts=None):
    from lcp_physics_b200.engines import engine_solve
    leaves = [soa[k].cuda().clone().requires_grad_(True) for k in NAMES]
    A = A0.clone().requires_grad_(True) if A0 is not None else None
    b = b0.clone().requires_grad_(True) if b0 is not None else None
    z, st = engine_solve(*leaves, b1, b2, DT, A=A, b=b, mode=mode, max_iter=max_iter, exact_adjoint=exact,
                         counts=counts)
    assert (st >= 0).all(), st.tolist()
    (z * gz).sum().backward()
    torch.cuda.synchronize()
    return _grads(leaves + ([A, b] if A0 is not None else []))


def _dense_grads(soa, b1, b2, A0, b0, mode, exact, gz, max_iter=5):
    from lcp_physics_b200 import LCPFunction
    from lcp_physics_b200.engines import assemble_contacts
    leaves = [soa[k].cuda().clone().requires_grad_(True) for k in NAMES]
    mass, inertia, v, fext, normal, p1, p2, mu, rest = leaves
    B, nc = mu.shape
    if A0 is not None:
        A, b = A0.clone().requires_grad_(True), b0.clone().requires_grad_(True)
    else:
        A = b = torch.tensor([], dtype=torch.float64, device="cuda")
    fn = LCPFunction(max_iter=max_iter, exact_adjoint=exact)
    if mode == 0:
        Q, p, G, h, F = assemble_contacts(mass, inertia, v, fext, normal, p1, p2, mu, rest, b1, b2, DT)
        z = fn(Q, p, G, h, A, b, F)
    else:                                                      # post_stabilization's LCP (engines.py:80-116)
        Q, _p, G, _h, _F = assemble_contacts(mass, inertia, v, fext, normal, p1, p2, mu, rest, b1, b2, 0.0)
        Jc = G[:, :nc, :].contiguous()
        jv = torch.bmm(Jc, v.unsqueeze(2)).squeeze(2)
        z = fn(Q, Q.new_zeros(B, Q.shape[1]), Jc, jv + jv * -rest, A, b, Q.new_zeros(B, nc, nc))
    (z * gz).sum().backward()
    torch.cuda.synchronize()
    return _grads(leaves + ([A, b] if A0 is not None else []))


@pytest.mark.parametrize("e", [0, 3])
@pytest.mark.parametrize("mode", [0, 1])
def test_fused_exact_adjoint_matches_dense_exact_adjoint(e, mode):
    B, nb, nc = 6, 8, 12
    soa = _soa_scene(B, nb, nc, seed=6)
    b1, b2 = soa["body1"].cuda(), soa["body2"].cuda()
    A0, b0 = _pins(B, e, 3 * nb) if e else (None, None)
    gz = torch.randn(B, 3 * nb, generator=torch.Generator().manual_seed(2), dtype=torch.float64).cuda()
    gf = _fused_grads(soa, b1, b2, A0, b0, mode, True, gz)
    gd = _dense_grads(soa, b1, b2, A0, b0, mode, True, gz)
    names = NAMES + (["A", "b"] if e else [])
    errs = {}
    for name, a, r in zip(names, gf, gd):
        assert torch.isfinite(a).all(), name
        errs[name] = float(rel_err(a.reshape(B, -1), r.reshape(B, -1)).max())
    # 5 iterations: away from the round-off floor of the KKT conditioning; 1e-4 = the fp64 gradient contract (DESIGN §5)
    assert max(errs.values()) < 1e-4, errs
    if mode == 0:
        # the flag reaches the kernel: with friction (F != 0) the reference's gradients are different ones
        gc = _fused_grads(soa, b1, b2, A0, b0, mode, False, gz)
        diff = {k: float(rel_err(gc[i].reshape(B, -1), gf[i].reshape(B, -1)).max()) for i, k in enumerate(NAMES)
                if k in ("mu", "v")}
        assert max(diff.values()) > 1e-3, diff


# ------------------------------------------------------------------ 2. banded vs condensed, exact flag
@pytest.mark.parametrize("e", [0, 3])
@pytest.mark.parametrize("mode", [0, 1])
def test_banded_exact_adjoint_matches_condensed(forced_banded, e, mode):
    B, nb, nc = 5, 16, 30
    soa = _soa_scene(B, nb, nc, seed=21)
    counts = torch.tensor([nc, nc - 7, nc, 11, nc - 1], dtype=torch.int32).cuda()
    b1 = soa["body1"].unsqueeze(0).expand(B, -1).contiguous().cuda()
    b2 = soa["body2"].unsqueeze(0).expand(B, -1).contiguous().cuda()
    A0, b0 = _pins(B, e, 3 * nb) if e else (None, None)
    gz = torch.randn(B, 3 * nb, dtype=torch.float64, generator=torch.Generator().manual_seed(3)).cuda()
    run = lambda exact: _fused_grads(soa, b1, b2, A0, b0, mode, exact, gz, max_iter=10, counts=counts)
    forced_banded(False)
    gcond = run(True)
    forced_banded(True)
    gband = run(True)
    errs = {}
    for name, gc, gb in zip(NAMES + ["A", "b"], gcond, gband):
        assert torch.isfinite(gb).all(), name
        errs[name] = float((gc - gb).norm() / gc.norm().clamp_min(1e-30)) if float(gc.norm()) > 0 else float(gb.norm())
    # the same contract and the same kappa(K) u as test_banded_backward_matches_condensed
    assert max(errs.values()) < 1e-4, errs
    gcompat = run(False)
    if mode == 1:
        # F = 0: W is a scalar per contact, the transposed system is the same one
        for name, a, c in zip(NAMES + ["A", "b"], gband, gcompat):
            assert torch.equal(a, c), name
    else:
        diff = max(float(rel_err(gcompat[i], gband[i]).max()) for i in (NAMES.index("mu"), NAMES.index("v")))
        assert diff > 1e-3, diff


# ------------------------------------------------------------------ 3. finite differences of one converged solve
def _fd_check(soa, b1, b2, A, b, counts, seed):
    from lcp_physics_b200.engines import engine_solve, last_solve_info
    B, n = soa["v"].shape
    gen = torch.Generator().manual_seed(seed)
    g = torch.randn(B, n, generator=gen, dtype=torch.float64).cuda()
    kw = dict(A=A, b=b, mode=0, max_iter=40, counts=counts)

    def loss(inp):
        z, st = engine_solve(*[inp[k].cuda() for k in NAMES], b1, b2, DT, **kw)
        assert (st >= 0).all()
        return (z * g).sum(1).cpu()

    grads = {}
    for exact in (True, False):
        leaves = [soa[k].cuda().clone().requires_grad_(True) for k in NAMES]
        z, st = engine_solve(*leaves, b1, b2, DT, exact_adjoint=exact, **kw)
        resid = last_solve_info()["resid"]
        assert (st >= 0).all() and float(resid.max()) < 1e-8, resid.tolist()   # converged: FD is a derivative
        (z * g).sum().backward()
        grads[exact] = dict(zip(NAMES, _grads(leaves)))
    valid = None
    if counts is not None:
        nc = soa["mu"].shape[1]
        valid = (torch.arange(nc).unsqueeze(0) < counts.cpu().unsqueeze(1)).to(torch.float64)
    h = 1e-5
    worst = {}
    for name in ("fext", "v", "mu", "restitution", "mass"):
        d = torch.randn(soa[name].shape, generator=gen, dtype=torch.float64)
        if valid is not None and name in ("mu", "restitution"):
            d = d * valid
        plus, minus = dict(soa), dict(soa)
        plus[name] = soa[name] + h * d
        minus[name] = soa[name] - h * d
        fd = (loss(plus) - loss(minus)) / (2 * h)
        scale = float(fd.abs().max())
        an = {ex: (grads[ex][name] * d).flatten(1).sum(1) for ex in (True, False)}
        worst[name] = tuple(float((an[ex] - fd).abs().max()) / scale for ex in (True, False))
    return worst


def _sliding_row(nballs, seed, dtype=torch.float64):
    """`nballs` balls (radius 10, 10 apart: they touch only the floor) resting on a pinned floor ball (body 0, radius
    1e5), all sliding the same way at 40 .. 60 and spinning, with friction 0.1 .. 0.4: the contact points still slide
    after 6 steps (friction slows them by at most 3 mu g = 120 per second) and the balls do not catch up with each
    other, so every complementarity pair stays strict and every solve converges far below 1e-8. nballs >= 43 gives
    n + e > 128: the banded kernel, with the floor (one contact per ball) and its pin in the border."""
    from lcp_physics_b200.scenes import make_ball_pile
    R, r = 1.0e5, 10.0
    ic = make_ball_pile(1, nballs=nballs, cols=nballs, seed=seed, gap=10.0, r=r, r_floor=R)
    dx = ic["pos"][:, 1:, 0] - 500.0
    ic["pos"][:, 1:, 1] = 500.0 + R - torch.sqrt((R + r + 0.05) ** 2 - dx * dx)   # 0.05 above the floor: in contact
    gen = torch.Generator().manual_seed(seed)
    ic["vel"][:, 1:, 1] = 40.0 + 20.0 * torch.rand(1, nballs, generator=gen, dtype=torch.float64)
    ic["vel"][:, 1:, 2] = 1.5                                  # towards the floor: restitution acts
    ic["vel"][:, 1:, 0] = torch.rand(1, nballs, generator=gen, dtype=torch.float64) - 0.5
    ic["fric"][:, 1:] = 0.1 + 0.3 * torch.rand(1, nballs, generator=gen, dtype=torch.float64)
    ic["rest"][:, 1:] = 0.2 + 0.5 * torch.rand(1, nballs, generator=gen, dtype=torch.float64)
    return {k: v.to(dtype) for k, v in ic.items()}, None


def _world_contact_soa(ic, cap):
    """The contact list of BatchedWorld(ic) at its initial state, as engine_solve inputs."""
    from lcp_physics_b200.world import BatchedWorld
    w = BatchedWorld(ic["pos"], ic["rad"], vel=ic["vel"], mass=ic["mass"], restitution=ic["rest"],
                     fric_coeff=ic["fric"], gravity=100.0, static=[0], dt=DT, contact_capacity=cap)
    soa = dict(mass=w.mass, inertia=w.inertia, v=w.v, fext=w.fext, normal=w.c_normal, p1=w.c_p1, p2=w.c_p2,
               mu=w.c_mu, restitution=w.c_rest)
    soa = {k: v.detach().cpu().clone() for k, v in soa.items()}
    return soa, w.c_b1, w.c_b2, w.A, torch.zeros(1, w.ne, dtype=torch.float64, device="cuda"), w.counts, w.large


@pytest.mark.parametrize("scene", ["soa_condensed", "soa_forced_banded", "row45_banded"])
def test_exact_adjoint_matches_finite_differences(forced_banded, scene):
    """Gradients of l = g . zhat of one converged engine solve (mode 0) against central differences along random
    directions of fext, v, mu, restitution and mass. worst[name] = (exact, bug-compatible) error relative to the
    FD scale. row45_banded: a 45-ball scene that selects the banded kernel by itself (pinned floor in the border,
    per-scene counts). The 60-ball piles of tests/golden/bworld_large.npz are not used: their solves stop at best
    residuals of 6e-8 .. 3e-7 (sticking and just-touching contacts), above the 1e-8 a difference quotient needs."""
    if scene == "row45_banded":
        soa, b1, b2, A, b, counts, large = _world_contact_soa(*_sliding_row(45, seed=3))
        assert large
        worst = _fd_check(soa, b1, b2, A, b, counts, seed=6)
    else:
        forced_banded(scene == "soa_forced_banded")
        soa = _soa_scene(4, 8, 12, seed=31)
        worst = _fd_check(soa, soa["body1"].cuda(), soa["body2"].cuda(), None, None, None, seed=5)
    # 2e-3: the gate of the dense API's FD check (test_exact_adjoint_matches_finite_differences_fp64)
    assert max(w[0] for w in worst.values()) < 2e-3, worst
    assert worst["mu"][1] > worst["mu"][0], worst


# ------------------------------------------------------------------ 4. BatchedWorld rollouts
INPUTS = ("vel", "fric", "rest")


def _rollout(ic, cap, leaves, wp, exact, steps=6):
    """wp . positions after `steps` steps of BatchedWorld(exact_adjoint=exact, max_iter=40, post_stab=False) from ic
    with (vel, fric_coeff, restitution) = leaves; also the per-step contact counts and times (the dt-halving history)
    and the largest best residual of every step's solve."""
    from lcp_physics_b200.engines import last_solve_info
    from lcp_physics_b200.world import BatchedWorld
    vel, fric, rest = leaves
    w = BatchedWorld(ic["pos"], ic["rad"], vel=vel, mass=ic["mass"], restitution=rest, fric_coeff=fric,
                     gravity=100.0, static=[0], dt=DT, max_iter=40, post_stab=False, contact_capacity=cap,
                     exact_adjoint=exact)
    hist, resid = [], []
    for _ in range(steps):
        w.step()
        hist.append((w.counts.tolist(), w.t.tolist()))
        resid.append(float(last_solve_info()["resid"].max()))
    return (w.p * wp.to(w.dtype)).sum(), hist, resid, w


def _rollout_grads(ic, cap, wp, exact):
    leaves = [ic[k].cuda().clone().requires_grad_(True) for k in INPUTS]
    loss, hist, resid, w = _rollout(ic, cap, leaves, wp, exact)
    loss.backward()
    torch.cuda.synchronize()
    return [t.grad.detach().cpu() for t in leaves], hist, resid, w


def rollout_fd_errors(ic, cap, seed=12, h=1e-5):
    """Exact and bug-compatible gradients of a 6-step rollout against central differences along one random direction
    per input: {name: (exact error, bug-compatible error)} relative to |FD|, with the history and residuals."""
    nb = ic["pos"].shape[1]
    gen = torch.Generator().manual_seed(seed)
    wp = torch.randn(1, nb, 3, generator=gen, dtype=torch.float64).cuda()
    ge, hist, resid, w = _rollout_grads(ic, cap, wp, True)
    gc, hist_c, _, _ = _rollout_grads(ic, cap, wp, False)
    assert hist_c == hist
    base = [ic[k].cuda() for k in INPUTS]
    errs = {}
    for i, name in enumerate(INPUTS):
        d = torch.randn(ic[name].shape, generator=gen, dtype=torch.float64)
        if name != "vel":
            d[:, 0] = 0                                        # the floor's coefficients: only the balls'
        with torch.no_grad():
            lp, hp, _, _ = _rollout(ic, cap, [t + h * d.cuda() if j == i else t for j, t in enumerate(base)], wp, True)
            lm, hm, _, _ = _rollout(ic, cap, [t - h * d.cuda() if j == i else t for j, t in enumerate(base)], wp, True)
        # identical contact sets and dt halving on both sides, or the difference quotient is not a derivative
        assert hp == hist and hm == hist, (name, hist, hp, hm)
        fd = float(lp - lm) / (2 * h)
        errs[name] = tuple(abs(float((g[i] * d).sum()) - fd) / abs(fd) for g in (ge, gc))
    return errs, hist, resid, w.large


@pytest.mark.parametrize("scene", ["row8_condensed", "row8_forced_banded", "row45_banded"])
def test_batched_world_exact_gradients_match_finite_differences(forced_banded, scene):
    """d(wp . positions after 6 steps) / d(initial vel, fric_coeff, restitution) through
    BatchedWorld(exact_adjoint=True) against central differences of the rollout. Every solve of the rollout must
    reach a best residual < 1e-8 (sliding contacts): only then is the rollout a differentiable map at the resolution
    of the difference quotient. errs[name] = (exact, bug-compatible) error relative to |FD|.

    Gate 2e-3, with one measured exception: restitution on the condensed kernel, 2e-2 (measured 1.4e-2). The
    restitution derivative is the smallest of the three here (it acts only through the balls' normal velocity), and
    the condensed fp64 backward carries more round-off than the banded one: the same rollout forced onto the banded
    kernel meets 2e-3 (measured 1.7e-4), and the reference's gradient is off by 4.5 along the same direction."""
    forced_banded(scene == "row8_forced_banded")
    nballs = 45 if scene == "row45_banded" else 8
    errs, hist, resid, large = rollout_fd_errors(*_sliding_row(nballs, seed=3))
    assert large == (scene == "row45_banded")
    assert max(resid) < 1e-8, resid
    assert all(c == [nballs] for c, _ in hist), hist         # every ball stays on the floor
    gate = {"vel": 2e-3, "fric": 2e-3, "rest": 2e-2 if scene == "row8_condensed" else 2e-3}
    assert all(errs[k][0] < gate[k] for k in gate), errs
    assert all(errs[k][1] > errs[k][0] for k in gate), errs  # the reference's gradients are worse along every one


def test_batched_world_fp32_exact_gradients_match_fp64():
    """The sliding-row rollout in fp32 (condensed kernels): exact gradients against the fp64 exact gradients, each
    relative to its own norm. vel and fric_coeff: 1e-3, the per-solve fp32 backward contract of DESIGN.md section 5
    (measured 1.1e-4 and 1.6e-5). restitution: 1e-2 (measured 5.5e-3): it acts only through the balls' normal
    velocity (1.5 against sliding speeds of 40 .. 60), so its gradient is a small sum of fp32 terms of the size of
    the others."""
    ic64, cap = _sliding_row(8, seed=3)
    wp = torch.randn(1, 9, 3, generator=torch.Generator().manual_seed(12), dtype=torch.float64).cuda()
    g64, h64, _, _ = _rollout_grads(ic64, cap, wp, True)
    g32, h32, _, _ = _rollout_grads({k: v.float() for k, v in ic64.items()}, cap, wp, True)
    assert [c for c, _ in h32] == [c for c, _ in h64], (h32, h64)
    errs = {name: float((a.double() - b).norm() / b.norm()) for name, a, b in zip(INPUTS, g32, g64)}
    assert errs["vel"] < 1e-3 and errs["fric"] < 1e-3 and errs["rest"] < 1e-2, errs


def test_batched_world_exact_adjoint_leaves_the_trajectory():
    """A 24-ball pile (sticking and just-touching contacts): the flag changes the gradients, never the trajectory."""
    from lcp_physics_b200.scenes import make_ball_pile
    ic = make_ball_pile(1, nballs=24, cols=6, seed=5, gap=0.05)
    ic["vel"][:, 1:] = torch.randn(1, 24, 3, generator=torch.Generator().manual_seed(9), dtype=torch.float64)
    wp = torch.randn(1, 25, 3, generator=torch.Generator().manual_seed(12), dtype=torch.float64).cuda()
    ge, he, _, we = _rollout_grads(ic, None, wp, True)
    gc, hc, _, wc = _rollout_grads(ic, None, wp, False)
    assert torch.equal(we.p, wc.p) and torch.equal(we.v, wc.v) and he == hc
    diff = {}
    for name, a, c in zip(INPUTS, ge, gc):
        assert torch.isfinite(a).all() and float(a.abs().max()) > 0, name
        diff[name] = float((a - c).norm() / c.norm())
    assert max(diff.values()) > 1e-3, diff


# ------------------------------------------------------------------ 5. B200PdipmEngine on recorded worlds
def _engine_grads(rec, fused, exact=True):
    from lcp_physics_b200.engines import B200PdipmEngine
    world = ReplayWorld(rec)
    world._v = world._v.clone().requires_grad_(True)
    for body in world.bodies:
        body.fric_coeff = torch.tensor(body.fric_coeff, dtype=torch.float64, requires_grad=True)
    eng = B200PdipmEngine(fused=fused, exact_adjoint=exact)
    out = eng.solve_dynamics(world, float(rec["dt"])) if str(rec["kind"]) == "solve_dynamics" else eng.post_stabilization(world)
    w = torch.randn(out.numel(), generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    (out.reshape(-1).cpu() * w).sum().backward()
    gf = torch.stack([b.fric_coeff.grad if b.fric_coeff.grad is not None else torch.zeros((), dtype=torch.float64)
                      for b in world.bodies])
    return world._v.grad.clone(), gf


@pytest.mark.parametrize("name", ["world_pile", "world_large"])
def test_engine_exact_adjoint_fused_matches_dense(name):
    """world_pile: condensed kernel fused, condensed dense; world_large (183 dofs): banded kernel fused, dual-form
    kernel dense. Gradients w.r.t. the replayed velocities and friction coefficients. Both paths must also differ
    from their own exact_adjoint=False gradients on the solve_dynamics calls (friction: F != 0), or the flag did not
    reach the kernels."""
    worst, moved = 0.0, {True: 0.0, False: 0.0}
    for rec in load_world_records(name):
        (vf, ff), (vd, fdn) = _engine_grads(rec, True), _engine_grads(rec, False)
        for a, r in ((vf, vd), (ff, fdn)):
            if float(r.norm()) == 0.0:
                assert float(a.norm()) == 0.0
                continue
            worst = max(worst, float((a - r).norm() / r.norm()))
        if str(rec["kind"]) == "solve_dynamics":
            for fused, (ve, fe) in ((True, (vf, ff)), (False, (vd, fdn))):
                vc, fc = _engine_grads(rec, fused, exact=False)
                moved[fused] = max(moved[fused], float((ve - vc).norm() / vc.norm()), float((fe - fc).norm() / fc.norm()))
    assert worst < 1e-4, worst
    assert min(moved.values()) > 1e-3, moved


def test_engine_exact_adjoint_refuses_a_replaced_solver():
    from lcp_physics_b200.engines import B200PdipmEngine

    class OtherSolver:                                         # e.g. the reference's LCPFunction
        def __init__(self, **kw):
            pass

        def __call__(self, *args):
            raise AssertionError("must not be reached")

    recs = {str(r["kind"]): r for r in load_world_records("world_pile")}
    eng = B200PdipmEngine(exact_adjoint=True)
    eng.lcp_solver = OtherSolver
    with pytest.raises(ValueError):
        eng.solve_dynamics(ReplayWorld(recs["solve_dynamics"]), float(recs["solve_dynamics"]["dt"]))
    with pytest.raises(ValueError):
        eng.post_stabilization(ReplayWorld(recs["post_stabilization"]))
