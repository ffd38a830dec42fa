"""GPU: the condensed-KKT kernels at every block count, component size and admission limit (DESIGN.md section 3.1).

Every result is compared with the CPU oracle (oracle/pdipm_oracle.py, fp64; the forward with per-scene semantics
and no pivoting).
Each test first proves which kernel ran: the plan's shared memory in `Handle.describe()` equals the host
restatement's (tests/cond_plan.py, whose verdicts for these scenes tests/test_cond_plan.py pins), a dense-API
scene's fallback to the dual form is read from the per-phase counters of a separate profiled call, and the engine
path reports it in `status`.

* every block count NS x dtype x {no equality rows, 3}: forward, both adjoints, structure reuse bitwise equal to
  rescanning; the engine path at NS = 8;
* component sizes 1 to 6 and a scene of mixed sizes;
* `comp_apply`'s whole grid: fp32 scenes with 129-150 five-row components (cfg 2's formulation on cfg 3's pile) and
  257-258 three-row components, whose last row slot lies past 4 positions per thread;
* each admission limit just inside (solved, matches the oracle) and just outside (bitwise the dual form's result on
  the dense API; status -100, no iterations and the other scenes unchanged on the engine path);
* per-scene contact counts 0, 1 and nc on the engine path, nc the most contacts the plan takes at 40 bodies.
"""
import numpy as np
import pytest
import torch

from tests import cond_plan as cp
from tests.helpers import dual_only, fp32_gate, rel_err

pytestmark = pytest.mark.gpu
GRADS = "dQ dp dG dh dA db dF".split()
ENGINE_NAMES = ["mass", "inertia", "v", "fext", "normal", "p1", "p2", "mu", "restitution"]
DT = 1.0 / 30
N_DUAL_PHASES = 14            # Handle.profile(): the dual-form phases come first


def _sizes(inp):
    Q, p, G, h, A, b, F = inp
    return Q.shape[1], G.shape[1], (A.shape[1] if A.dim() > 1 else 0)


def _handle(dtype, n, m, e):
    from lcp_physics_b200 import _lib
    return _lib.get_handle(dtype, n, m, e, torch.cuda.current_device(), torch.cuda.current_stream().cuda_stream)


def _check_plan(dtype, n, m, e):
    """The plan the library made is the restatement's (same shared memory and CTAs per SM)."""
    plan = cp.make_plan(cp.tsize(dtype), n, m, e)
    desc = _handle(dtype, n, m, e).describe()
    if plan is None:
        assert "condensed KKT: n/a" in desc, desc
    else:
        assert "smem=%dB CTAs/SM=%d" % (plan["smem_bytes"], plan["ctas_per_sm"]) in desc, (plan, desc)
    return plan


def _dual_ran(inp, dtype):
    """Whether the dual-form forward kernel solved any scene: a profiled call (its own instantiation; its results
    are not compared) whose dual-form phase counters stay zero unless some scene was flagged -100."""
    from lcp_physics_b200 import solve_forward
    n, m, e = _sizes(inp)
    hd = _handle(dtype, n, m, e)
    hd.profile(True)
    solve_forward(*[t.to(dtype).cuda() for t in inp], max_iter=2)
    torch.cuda.synchronize()
    prof = list(hd.profile(False).values())
    return sum(prof[:N_DUAL_PHASES]) > 0


def _forward(inp, dtype, max_iter=10, save=None):
    from lcp_physics_b200 import solve_forward
    out = solve_forward(*[t.to(dtype).cuda() for t in inp], max_iter=max_iter, save=save)
    torch.cuda.synchronize()
    return out


def _oracle(inp, max_iter=10):
    from oracle import pdipm_oracle as po
    return po.lcp_forward(*inp, max_iter=max_iter, coupled=False, pivot=False)


def _gz(B, n, seed=3):
    return torch.randn(B, n, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


def _check_forward(inp, dtype, B_gate=None):
    """Forward against the oracle: fp64 zhat at 1e-6; fp32 per scene after one iteration (the initial point:
    zhat, lam and slack of one KKT solve, not chaotic) and the distribution gate after 10."""
    if dtype == torch.float64:
        out = _forward(inp, dtype)
        assert (out[4] >= 0).all()
        assert rel_err(out[0].cpu(), _oracle(inp).zhat).max() < 1e-6
        return out
    one, ref1 = _forward(inp, dtype, max_iter=1), _oracle(inp, max_iter=1)
    for k, name in ((0, "zhat"), (2, "lam"), (3, "slack")):
        err = rel_err(one[k].cpu(), getattr(ref1, {"zhat": "zhat", "lam": "lams", "slack": "slacks"}[name]))
        assert err.max() < 1e-4, (name, err)
    out = _forward(inp, dtype)
    assert (out[4] >= 0).all()
    ref64 = _oracle(inp).zhat
    if B_gate:
        fp32_gate(out[0].cpu(), _oracle([t.float() for t in inp]).zhat, ref64, "fp32")
    else:
        # after 10 iterations fp32 trajectories are chaotic on a few per cent of the scenes (test_gpu_parity's
        # docstring): too few scenes here for the distribution gate, so a median and a loose bound
        err = rel_err(out[0].cpu(), ref64)
        assert err.median() < 1e-3 and err.max() < 5e-2, err
    return out


def _check_backward(inp, dtype, g):
    """Both adjoints against the oracle on the same forward state; the structure the forward saved gives bitwise the
    gradients of a rescan. fp64 (the dual form's backward, the condensed kernel as its rescue): the kernel's own state,
    dlam / dnu (dG, dh, dF, dA, db) are noise on scenes at the round-off floor. fp32 (the condensed backward): the
    oracle's state after 5 iterations, rounded to fp32, away from the fp32 floor where any fp32 backward loses digits."""
    from lcp_physics_b200 import solve_backward
    from oracle import pdipm_oracle as po
    n, m, e = _sizes(inp)
    Q, p, G, h, A, b, F = [t.to(dtype).cuda() for t in inp]
    saved = {}
    zhat, nu, lam, slack = _forward(inp, dtype, save=saved)[:4]
    if dtype == torch.float32:
        r = _oracle(inp, max_iter=5)
        zhat, lam, slack = (t.to(dtype).cuda() for t in (r.zhat, r.lams, r.slacks))
        nu = r.nus.to(dtype).cuda() if e else None
    gd = g.to(dtype).cuda()
    state = [zhat.double().cpu(), nu.double().cpu() if e else None, lam.double().cpu(), slack.double().cpu()]
    floor = (torch.minimum(state[3].min(1)[0], state[2].min(1)[0]) < 1e-12)
    for exact, ora in ((False, po.lcp_backward_from_saved), (True, po.lcp_backward_exact_from_saved)):
        reused = solve_backward(Q, G, A, F, zhat, nu, lam, slack, gd, saved=saved, exact_adjoint=exact)
        scanned = solve_backward(Q, G, A, F, zhat, nu, lam, slack, gd, exact_adjoint=exact)
        truth = ora(inp, *state, g)
        for name, a, c, t in zip(GRADS, reused, scanned, truth):
            if t is None:
                assert a is None and c is None
                continue
            assert torch.equal(a, c), (name, exact)
            assert torch.isfinite(a).all(), (name, exact)
            err = rel_err(a.cpu(), t)
            if dtype == torch.float64:
                if name in ("dG", "dh", "dF", "dA", "db"):       # dlam, dnu: KKT noise at the round-off floor
                    err = err[~floor]
                if err.numel():
                    assert err.max() < 1e-3 and err.median() < 1e-5, (name, exact, err)
            else:
                assert err.max() < 1e-3 and err.median() < 1e-4, (name, exact, err)


# ------------------------------------------------------------------ every block count, dense API
NS_SCENES = {2: (8, 16), 3: (14, 28), 4: (20, 40), 6: (30, 60), 8: (40, 80)}      # NS: (bodies, contacts)


@pytest.mark.parametrize("e", [0, 3])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("NS", sorted(NS_SCENES))
def test_every_block_count_dense_api(NS, dtype, e):
    nb, nc = NS_SCENES[NS]
    B = 4
    inp = cp.contact_scenes(B, nb, nc, 2, e=e, seed=40 + NS)
    n, m, _ = _sizes(inp)
    plan = _check_plan(dtype, n, m, e)
    assert plan["NS"] == NS
    assert not _dual_ran(inp, dtype)
    _check_forward(inp, dtype)
    _check_backward(inp, dtype, _gz(B, n))


# ------------------------------------------------------------------ component sizes 1 .. 6 and mixed sizes
CS_SCENES = {   # name: (builder, cs)
    "cs1_poststab": (lambda: cp.poststab_scenes(4, 16, 32, seed=51), 1),
    "cs2_monotone_block": (lambda: cp.cs2_scenes(4, 16, 32, seed=52), 2),
    "cs3_fd1": (lambda: cp.contact_scenes(4, 16, 32, 1, seed=53), 3),
    "cs4_fd2": (lambda: cp.contact_scenes(4, 16, 32, 2, seed=54), 4),
    "cs5_fd3": (lambda: cp.contact_scenes(4, 16, 32, 3, seed=55), 5),
    "cs6_fd4": (lambda: cp.contact_scenes(4, 16, 32, 4, seed=56), 6),
    "mixed_4_and_1": (lambda: cp.mixed_scenes(4, 16, 32, seed=57), 4),
}


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("name", list(CS_SCENES))
def test_every_component_size(name, dtype):
    """fp32: forward and both adjoints run on the condensed kernels; fp64: the forward does (the fp64 backward
    takes the dual form first)."""
    build, cs = CS_SCENES[name]
    inp = build()
    n, m, e = _sizes(inp)
    plan = _check_plan(dtype, n, m, e)
    v = cp.verdict_dense(inp[0][0], inp[2][0], inp[6][0], e, plan)
    assert v["ok"] and v["cs"] == cs, v
    assert not _dual_ran(inp, dtype)
    _check_forward(inp, dtype)
    _check_backward(inp, dtype, _gz(inp[0].shape[0], n))


# ------------------------------------------------------------------ comp_apply's whole grid
def test_five_row_components_past_four_positions_per_thread():
    """cfg 2's formulation (3 friction directions) on cfg 3's 8 x 4 pile with 140 contacts: 140 components of 5 rows,
    sh = 8, so comp_apply's grid is 5 << 8 = 1280 positions, 5 per thread. With 4 per thread the gamma rows (slot 4)
    were never multiplied by W_c: dz, ds and everything after them were wrong."""
    from lcp_physics_b200.scenes import make_scenes
    B = 12
    inp = make_scenes(B, 32, 140, fd=3, e=0, dtype=torch.float64, seed=61)
    n, m, e = _sizes(inp)
    plan = _check_plan(torch.float32, n, m, e)
    v = cp.verdict_dense(inp[0][0], inp[2][0], inp[6][0], 0, plan)
    assert v["ok"] and (v["ncomp"], v["cs"], v["sh"]) == (140, 5, 8) and not cp.apply_grid_ok(v, old=True), v
    assert not _dual_ran(inp, torch.float32)
    _check_forward(inp, torch.float32, B_gate=True)
    _check_backward(inp, torch.float32, _gz(B, n))


def test_three_row_components_past_four_positions_per_thread():
    """257 one-body contacts with one friction direction on 20 bodies (n = 60): 257 components of 3 rows, sh = 9,
    a grid of 3 << 9 = 1536 positions (6 per thread). Only one-body rows fit 257 components into the 16 list
    entries per column at this n."""
    sc = cp.floor_contacts(20, 257)
    inp = cp.dense_from_graph(sc, 4, 1, seed=62)
    n, m, e = _sizes(inp)
    plan = _check_plan(torch.float32, n, m, e)
    v = cp.verdict_dense(inp[0][0], inp[2][0], inp[6][0], 0, plan)
    assert v["ok"] and (v["ncomp"], v["cs"], v["sh"]) == (257, 3, 9) and not cp.apply_grid_ok(v, old=True), v
    assert not _dual_ran(inp, torch.float32)
    one, ref1 = _forward(inp, torch.float32, max_iter=1), _oracle(inp, max_iter=1)
    for k, name in ((0, "zhat"), (2, "lams"), (3, "slacks")):
        err = rel_err(one[k].cpu(), getattr(ref1, name))
        assert err.max() < 1e-4, (name, err)


# ------------------------------------------------------------------ admission limits, dense API
@pytest.mark.parametrize("limit", list(cp.LIMIT_SCENES))
def test_dense_admission_limit(limit):
    """Just inside: the condensed kernel solves the scene and matches the oracle. Just outside: the scene's outputs
    are bitwise those of a dual-form run."""
    dtype, inside, outside = cp.limit_scenes(limit)
    for inp, ok in ((inside, True), (outside, False)):
        n, m, e = _sizes(inp)
        plan = _check_plan(dtype, n, m, e)
        v = cp.verdict_dense(inp[0][0], inp[2][0], inp[6][0], e, plan)
        assert v["ok"] == ok, (limit, v)
        if plan is not None:
            assert _dual_ran(inp, dtype) == (not ok), limit
        if ok:
            _check_forward(inp, dtype)
        else:
            out = _forward(inp, dtype)
            with dual_only():
                ref = _forward(inp, dtype)
            for a, b in zip(out, ref):
                if a is not None:
                    assert torch.equal(a, b), limit


# ------------------------------------------------------------------ engine path
def _engine(soa, dtype, mode=0, counts=None, exact=False, g=None, A=None, b=None):
    from lcp_physics_b200.engines import engine_solve, last_solve_info
    leaves = [soa[k].to(dtype).cuda().requires_grad_(True) for k in ENGINE_NAMES]
    b1, b2 = soa["body1"].cuda(), soa["body2"].cuda()
    z, st = engine_solve(*leaves, b1, b2, DT, A=A, b=b, mode=mode, max_iter=10, exact_adjoint=exact,
                         counts=None if counts is None else counts.cuda())
    info = {k: (v.clone() if v is not None else None) for k, v in last_solve_info().items()}
    if g is not None:
        (z * g.to(dtype).cuda()).sum().backward()
    torch.cuda.synchronize()
    return z, st, info, [t.grad for t in leaves]


def _engine_dense(soa, counts=None):
    """The engine's LCP per scene as dense fp64 inputs (assemble_dense on each scene's own contacts)."""
    from lcp_physics_b200.scenes import assemble_dense
    B = soa["mass"].shape[0]
    out = []
    for s in range(B):
        k = soa["body1"].shape[-1] if counts is None else int(counts[s])
        one = {}
        for name, t in soa.items():
            if name in ("body1", "body2"):
                one[name] = (t[s] if t.dim() == 2 else t)[:k]
            elif name in ("mass", "inertia", "v", "fext"):
                one[name] = t[s:s + 1]
            else:
                one[name] = t[s:s + 1, :k]
        inp = assemble_dense(one, fd=2)
        fext = one["fext"]
        Md = torch.stack([one["inertia"], one["mass"], one["mass"]], -1).reshape(1, -1)
        inp = (inp[0], Md * one["v"] + DT * fext) + inp[2:]
        out.append(inp)
    return out


def _engine_vs_oracle(soa, dtype, counts=None):
    """Forward and both adjoints of the engine path against per-scene dense oracle solves."""
    from oracle import pdipm_oracle as po
    B, nb = soa["mass"].shape
    g = _gz(B, 3 * nb, seed=9)
    per = _engine_dense(soa, counts)
    for exact in (False, True):
        z, st, info, grads = _engine(soa, dtype, counts=counts, exact=exact, g=g)
        assert (st == 2).all() or (st >= 0).all()
        for s, inp in enumerate(per):
            if inp[2].shape[1] == 0:          # no contacts: Q zhat + p = 0
                want = -inp[1] / torch.diagonal(inp[0], dim1=1, dim2=2)
                assert rel_err(z[s:s + 1].detach().cpu(), want).max() < (1e-12 if dtype == torch.float64 else 1e-6)
                continue
            ref = _oracle(inp)
            tol = 1e-6 if dtype == torch.float64 else 2e-2
            assert rel_err(z[s:s + 1].detach().cpu(), ref.zhat).max() < tol, (s, exact)
            ora = po.lcp_backward_exact_from_saved if exact else po.lcp_backward_from_saved
            dp = ora(inp, z[s:s + 1].detach().double().cpu(), None, info["lam"][s:s + 1, :inp[2].shape[1]].double().cpu(),
                     info["slack"][s:s + 1, :inp[2].shape[1]].double().cpu(), g[s:s + 1], pivot=False)[1]
            # dp = dx: the engine's dfext is dt dx
            got = grads[3][s:s + 1].detach().double().cpu() / DT
            assert rel_err(got, dp).max() < (1e-4 if dtype == torch.float64 else 1e-3), (s, exact)
    return z, st


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("nb", [36, 40])
def test_engine_path_at_eight_blocks(nb, dtype):
    from lcp_physics_b200.scenes import make_contact_soa
    soa = dict(make_contact_soa(3, nb, 2 * nb, seed=70 + nb))
    fext = torch.zeros(3, 3 * nb, dtype=torch.float64)
    fext[:, 2::3] = 10.0 * soa["mass"]
    soa["fext"] = fext
    plan = _check_plan(dtype, 3 * nb, 8 * nb, 0)
    assert plan["NS"] == 8
    _engine_vs_oracle(soa, dtype)


@pytest.mark.parametrize("dtype,nc", [(torch.float64, 108), (torch.float32, 176)])
def test_engine_per_scene_counts_and_largest_m(dtype, nc):
    """Contact counts 0, 1 and nc in one batch, nc the most contacts of 40 bodies the condensed plan takes (the
    shared memory binds before m = 1024 does), each scene against its own dense oracle solve."""
    sc = cp.circulant(40, nc)
    soa = cp.graph_soa(sc, 3, seed=71)
    plan = _check_plan(dtype, 120, 4 * nc, 0)
    assert plan is not None and plan["NS"] == 8
    counts = torch.tensor([0, 1, nc], dtype=torch.int32)
    soa["body1"] = soa["body1"].unsqueeze(0).expand(3, -1).contiguous()
    soa["body2"] = soa["body2"].unsqueeze(0).expand(3, -1).contiguous()
    z, st = _engine_vs_oracle(soa, dtype, counts=counts)
    assert int(st[0]) == 2


def test_engine_column_limit_hub():
    """A hub with 16 contacts is solved; with 17 its scene gets status -100 and no iterations, and the other scenes of
    the batch are bitwise what they are without it. B200PdipmEngine then falls back to the dense path."""
    import copy
    ok_sc, bad_sc = cp.bp.hubs(1, 16, ring=40), cp.bp.hubs(1, 17, ring=40)
    for sc, ok in ((ok_sc, True), (bad_sc, False)):
        nc = len(sc["body1"])
        plan = cp.make_plan(8, 3 * sc["nb"], 4 * nc, 0)
        v = cp.verdict_soa(sc["nb"], sc["body1"], sc["body2"], nc, 0, 0, plan)
        assert v["ok"] == ok and (ok or v["rule"] == "LMAX"), v
    # per-scene topologies: scene 1 has the 17th hub contact, scenes 0 and 2 use the same slot for a ring contact
    nb, nc = bad_sc["nb"], len(bad_sc["body1"])
    soa = cp.graph_soa(bad_sc, 3, seed=72)
    b1 = soa["body1"].unsqueeze(0).repeat(3, 1)
    b2 = soa["body2"].unsqueeze(0).repeat(3, 1)
    last = nc - 1
    assert int(b1[0, last]) == 0 or int(b2[0, last]) == 0
    b1[[0, 2], last], b2[[0, 2], last] = 5, 6
    soa["body1"], soa["body2"] = b1, b2
    counts = torch.full((3,), nc, dtype=torch.int32)                 # per-scene contact lists
    for dtype in (torch.float64, torch.float32):
        z, st, info, _ = _engine(soa, dtype, counts=counts)
        assert st.tolist()[1] == -100 and int(info["iters"][1]) == 0 and st[0] >= 0 and st[2] >= 0, st
        alone = copy.deepcopy(soa)
        for k in alone:
            alone[k] = alone[k][[0, 2]]
        z2, st2, _, _ = _engine(alone, dtype, counts=counts[:2])
        assert torch.equal(z[[0, 2]], z2)
    # the reference-style engine on a world with the degree-17 hub: dense fallback, against the oracle
    from lcp_physics_b200.engines import B200PdipmEngine
    from tests.helpers import ReplayWorld
    rec, inp = cp.hub_world_record(bad_sc, seed=73)
    new_v = B200PdipmEngine().solve_dynamics(ReplayWorld(rec), DT)
    assert rel_err(-new_v.detach().double().cpu().reshape(1, -1), _oracle(inp).zhat).max() < 1e-6
