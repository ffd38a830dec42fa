"""GPU: forward-mode derivatives (Jacobian-vector products) through the engine solve and BatchedWorld.

1. The kernel JVP (lcpb200_engine_jvp_batched through torch.func.jvp) equals an independent dense fp64 solve of the
   linearised KKT system at the saved iterate, on condensed and forced-banded scenes, both LCP modes, with and
   without equality rows, with a zero-contact scene; the status -100 scene gets zero rows.
2. jacfwd equals jacrev with the exact adjoint (condensed, forced banded, a natural banded pile) and central
   differences on converged solves; fp32 against fp64.
3. One jacfwd call with R tangents equals R torch.func.jvp calls: bitwise on the condensed kernels, 1e-10 on the
   banded one; forward_ad dual tensors give bitwise what torch.func.jvp gives.
4. jacfwd of a BatchedWorld step equals linearize() with the exact adjoint; tangents through obstacle vertices and
   polygon poses are non-zero and match central differences (the contact geometry follows the tangents).
5. Rollout sensitivities w.r.t. friction, mass and initial velocity: forward against reverse mode and central
   differences; the forward-mode rollout's peak memory does not grow with its length.
"""
import pytest
import torch
import torch.autograd.forward_ad as fwAD

from tests.test_gpu_jacobians import (DT, _pile60, _polygon_bin, _rel, _row_scale_err, _scene, _sliding_balls,
                                      _soa_case, _solve_fn, _step_from, _world_soa,
                                      forced_banded)   # noqa: F401  (forced_banded: a fixture)

pytestmark = pytest.mark.gpu
f64 = torch.float64


def _tangents(args, R, seed, dtype):
    """Random tangents [R, *shape] for every input; normals stay on the unit circle to first order."""
    gen = torch.Generator().manual_seed(seed)
    out = []
    for i, t in enumerate(args):
        d = torch.randn((R,) + tuple(t.shape), generator=gen, dtype=f64).to(dtype).cuda()
        if i == 4:
            d = d - (d * t).sum(-1, keepdim=True) * t
        out.append(d)
    return out


# ------------------------------------------------------------------ 1. dense reference
def _dense_lcp(mass, inertia, v, fext, normal, p1, p2, mu, rest, b1, b2, nc, mode):
    """Q, p, G, h, F of ONE scene with its first nc contacts, in torch (world.py:144-234, engines.py:50-116)."""
    nb = mass.shape[0]
    n = 3 * nb
    q = torch.stack([inertia, mass, mass], 1).reshape(n)
    Q = torch.diag(q)

    def rows(d):
        R = normal.new_zeros(nc, n)
        for c in range(nc):
            i, j = int(b1[c]), int(b2[c])
            R[c, 3 * i:3 * i + 3] = torch.stack([p1[c, 0] * d[c, 1] - p1[c, 1] * d[c, 0], d[c, 0], d[c, 1]])
            if j < nb:
                R[c, 3 * j:3 * j + 3] = -torch.stack([p2[c, 0] * d[c, 1] - p2[c, 1] * d[c, 0], d[c, 0], d[c, 1]])
        return R
    nrm = normal[:nc]
    Jc = rows(nrm)
    jv = Jc @ v
    if mode == 1:
        return Q, torch.zeros_like(v), Jc, jv * (1 - rest[:nc]), normal.new_zeros(nc, nc)
    Jf1 = rows(torch.stack([nrm[:, 1], -nrm[:, 0]], 1))
    Jf = torch.stack([Jf1, -Jf1], 1).reshape(2 * nc, n)
    G = torch.cat([Jc, Jf, normal.new_zeros(nc, n)])
    h = torch.cat([jv * rest[:nc], normal.new_zeros(3 * nc)])
    E = torch.zeros(2 * nc, nc, dtype=normal.dtype, device=normal.device)
    E[torch.arange(2 * nc), torch.arange(nc).repeat_interleave(2)] = 1
    Z = lambda r, c: normal.new_zeros(r, c)
    F = torch.cat([torch.cat([Z(nc, nc), Z(nc, 2 * nc), Z(nc, nc)], 1),
                   torch.cat([Z(2 * nc, nc), Z(2 * nc, 2 * nc), E], 1),
                   torch.cat([torch.diag(mu[:nc]), -E.t(), Z(nc, nc)], 1)])
    return Q, q * v + DT * fext, G, h, F


def _dense_jvp(prim, tan, b1, b2, nc, mode, zhat, lam, slack, nu):
    """Tangent of zhat from the linearised KKT system K [dx; ds; dz; dy] = -(r_x, 0, r_z, r_y) at the saved iterate,
    d = lam / slack clamped to [1e-10, 1e10], the dense assembly differentiated by torch.func.jvp."""
    (Q, p, G, h, F), (dQ, dp, dG, dh, dF) = torch.func.jvp(
        lambda *x: _dense_lcp(*x, b1, b2, nc, mode), tuple(prim[:9]), tuple(tan[:9]))
    A, dA, db = prim[9], tan[9], tan[10]
    n, m = Q.shape[0], G.shape[0]
    e = 0 if A is None else A.shape[0]
    z, lm = zhat, lam[:m]
    rx = dQ @ z + dp + dG.t() @ lm
    rz = dG @ z - dF @ lm - dh
    if e:
        rx = rx + dA.t() @ nu
        ry = dA @ z - db
    d = (lm / slack[:m]).clamp(1e-10, 1e10)
    # ds = -dz / d (the complementarity row, rs = 0) eliminated: [[Q, G^T, A^T], [G, -(F + 1/d), 0], [A, 0, 0]]
    # [dx; dz; dy] = -(r_x, r_z, r_y), rows and columns of dz scaled by min(1, sqrt(d)) so that the 1/d of inactive
    # rows (up to 1e10) does not set the condition number
    N = n + m + e
    K = Q.new_zeros(N, N)
    K[:n, :n] = Q
    K[:n, n:n + m] = G.t()
    K[n:n + m, :n] = G
    K[n:n + m, n:n + m] = -(F + torch.diag(1 / d))
    rhs = torch.cat([rx, rz])
    if e:
        K[n + m:, :n] = A
        K[:n, n + m:] = A.t()
        rhs = torch.cat([rhs, ry])
    sc = torch.ones(N, dtype=f64, device=Q.device)
    sc[n:n + m] = d.sqrt().clamp_max(1.0)
    y = torch.linalg.solve(sc[:, None] * K * sc[None, :], -sc * rhs)
    return (sc * y)[:n]


@pytest.mark.parametrize("e", [0, 3])
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("kernel", ["condensed", "forced_banded"])
def test_kernel_jvp_matches_dense_linearised_kkt(forced_banded, kernel, mode, e):
    from lcp_physics_b200.engines import assemble_contacts, last_solve_info
    forced_banded(kernel == "forced_banded")
    nb, nc, B = (6, 8, 5) if kernel == "condensed" else (16, 30, 5)
    ins, A, b, b1, b2, counts = _soa_case(B, nb, nc, e, f64, seed=13, special=True)
    counts[3] = nc // 2                                                  # a scene with a shorter contact list
    args = ins + ([A, b] if e else [])
    f = _solve_fn(b1, b2, mode, False, counts, e)
    tan = [t[0] for t in _tangents(args, 1, seed=5, dtype=f64)]
    zhat, dz = torch.func.jvp(f, tuple(args), tuple(tan))
    info = last_solve_info()
    st = info["status"]
    assert int(st[2]) == -100 and (st[[0, 1, 3, 4]] >= 0).all(), st.tolist()
    assert not dz[2].any()
    for s in (0, 1, 3, 4):
        k = int(counts[s])
        sl = lambda xs: [x[s] for x in xs]
        prim, tg = sl(ins), sl(tan[:9])
        if s == 0 and mode == 0:                                         # the torch assembly is the kernel's
            Qa, pa, Ga, ha, Fa = assemble_contacts(*[x[s:s + 1] for x in ins[:7]], ins[7][s:s + 1], ins[8][s:s + 1],
                                                   b1[s].contiguous(), b2[s].contiguous(), DT)
            Qd, pd, Gd, hd, Fd = _dense_lcp(*prim, b1[s], b2[s], k, 0)
            for x, y in ((Qa, Qd), (pa, pd), (Ga, Gd), (ha, hd), (Fa, Fd)):
                assert torch.allclose(x[0], y, rtol=1e-13, atol=1e-13)
        prim += [A[s], b[s]] if e else [None, None]
        tg += [tan[9][s], tan[10][s]] if e else [None, None]
        ref = _dense_jvp(prim, tg, b1[s], b2[s], k, mode, zhat[s], info["lam"][s], info["slack"][s],
                         info["nu"][s] if e else None)
        err = float((dz[s] - ref).abs().max()) / max(float(ref.abs().max()), 1e-12)   # mode 1, no row: zhat = 0
        # the kernels solve the condensed system K = Q + G^T W G; at a converged iterate d = lam / s sits at its clamp
        # (1e+-10), W reaches 1e10 and K's round-off is ~1e-6 of the result (the backward shares it)
        assert err <= 3e-5, (s, err)


# ------------------------------------------------------------------ 2. forward against reverse mode
WHICH = {"mass": 0, "inertia": 1, "v": 2, "fext": 3, "normal": 4, "p1": 5, "p2": 6, "mu": 7, "restitution": 8, "A": 9}


def _converged_case(scene, forced_banded, dtype=f64):
    forced_banded(scene == "row8_forced_banded")
    if scene == "pile60_banded":
        w = _pile60()
        w.step()
    else:
        w = _sliding_balls(1, 45 if scene == "row45_banded" else 8, seed=3, dtype=dtype)
    ins = _world_soa(w)
    A, b = w.A.detach().clone(), torch.zeros(1, w.ne, dtype=dtype, device="cuda")
    return w, ins + [A, b]


@pytest.mark.parametrize("scene", ["row8_condensed", "row8_forced_banded", "row45_banded", "pile60_banded"])
def test_jacfwd_equals_exact_jacrev(forced_banded, scene):
    w, args = _converged_case(scene, forced_banded)
    assert w.large == (scene in ("row45_banded", "pile60_banded"))
    argnums = tuple(WHICH.values())
    Jf = torch.func.jacfwd(_solve_fn(w.c_b1, w.c_b2, 0, False, w.counts, w.ne, max_iter=40), argnums=argnums)(*args)
    Jr = torch.func.jacrev(_solve_fn(w.c_b1, w.c_b2, 0, True, w.counts, w.ne, max_iter=40), argnums=argnums)(*args)
    n = 3 * w.nd
    top = max(float(j.abs().max()) for j in Jr)
    errs = {}
    for name, x, y in zip(WHICH, Jf, Jr):
        # against the largest entry of this input's Jacobian: K and K^T are solved separately, each carrying the
        # condensed system's round-off at a converged iterate (test_kernel_jvp_matches_dense_linearised_kkt)
        errs[name] = float((x - y).abs().max()) / max(float(y.abs().max()), 1e-12 * top)
    assert max(errs.values()) <= 1e-4, errs


@pytest.mark.parametrize("scene", ["row8_condensed", "row8_forced_banded", "row45_banded"])
def test_jvp_matches_finite_differences(forced_banded, scene):
    """One converged solve (residual < 1e-8): the JVP along a random direction of each input against central
    differences, as test_jacrev_matches_finite_differences does for the VJP."""
    from lcp_physics_b200.engines import last_solve_info
    w, args = _converged_case(scene, forced_banded)
    f = _solve_fn(w.c_b1, w.c_b2, 0, False, w.counts, w.ne, max_iter=40)
    f(*args)
    assert float(last_solve_info()["resid"].max()) < 1e-8
    gen = torch.Generator().manual_seed(7)
    h = 1e-6
    worst, scale = {}, {}
    for name, i in WHICH.items():
        d = torch.randn(args[i].shape, generator=gen, dtype=f64).cuda()
        if name == "normal":
            d = d - (d * args[i]).sum(-1, keepdim=True) * args[i]
        if name == "A":
            d = d * (args[i] != 0).any(1, keepdim=True)
        tan = [d if j == i else torch.zeros_like(t) for j, t in enumerate(args)]
        _, an = torch.func.jvp(f, tuple(args), tuple(tan))
        plus = [t + h * d if j == i else t for j, t in enumerate(args)]
        minus = [t - h * d if j == i else t for j, t in enumerate(args)]
        fd = (f(*plus) - f(*minus)) / (2 * h)
        worst[name], scale[name] = float((an - fd).abs().max()), float(fd.abs().max())
    top = max(scale.values())
    rel = {k: worst[k] / (scale[k] if scale[k] > 1e-6 * top else top) for k in worst}
    assert max(rel.values()) < 1e-4, sorted(rel.items(), key=lambda kv: -kv[1])


def test_jacfwd_fp32_matches_fp64(forced_banded):
    w64, a64 = _converged_case("row8_condensed", forced_banded)
    w32, a32 = _converged_case("row8_condensed", forced_banded, dtype=torch.float32)
    argnums = tuple(WHICH.values())
    J64 = torch.func.jacfwd(_solve_fn(w64.c_b1, w64.c_b2, 0, False, w64.counts, w64.ne, max_iter=40), argnums=argnums)(*a64)
    J32 = torch.func.jacfwd(_solve_fn(w32.c_b1, w32.c_b2, 0, False, w32.counts, w32.ne, max_iter=40), argnums=argnums)(*a32)
    top = max(float(j.abs().max()) for j in J64)
    for name, x, y in zip(WHICH, J32, J64):
        assert x.dtype == torch.float32
        assert float((x.double() - y).abs().max()) <= 1e-3 * max(float(y.abs().max()), 1e-3 * top), name


# ------------------------------------------------------------------ 3. batching
def _batched_and_sequential_jvp(ins, A, b, b1, b2, counts, mode, R, seed):
    e = 0 if A is None else A.shape[1]
    f = _solve_fn(b1, b2, mode, False, counts, e)
    args = ins + ([A, b] if e else [])
    T = _tangents(args, R, seed, ins[0].dtype)
    batched = torch.func.vmap(lambda *t: torch.func.jvp(f, tuple(args), t)[1])(*T)
    seq = torch.stack([torch.func.jvp(f, tuple(args), tuple(t[r] for t in T))[1] for r in range(R)])
    with fwAD.dual_level():
        dual = fwAD.unpack_dual(f(*[fwAD.make_dual(x, t[0]) for x, t in zip(args, T)])).tangent
    from lcp_physics_b200.engines import last_solve_info
    return batched, seq, dual, last_solve_info()["status"]


@pytest.mark.parametrize("B", [4, 300])                 # 4: several chunks of tangents per scene; 300: one
@pytest.mark.parametrize("R", [1, 7, "n"])
@pytest.mark.parametrize("e", [0, 3])
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_condensed_batched_jvp_equals_sequential(dtype, mode, e, R, B):
    nb, nc = 6, 8
    ins, A, b, b1, b2, counts = _soa_case(B, nb, nc, e, dtype, seed=3, special=True)
    R = 3 * nb if R == "n" else R
    batched, seq, dual, status = _batched_and_sequential_jvp(ins, A, b, b1, b2, counts, mode, R, seed=R + B)
    assert int(status[2]) == -100 and int(status[1]) >= 0, status.tolist()
    assert batched.shape == (R, B, 3 * nb)
    assert torch.equal(batched, seq), float((batched - seq).abs().max())
    assert torch.equal(dual, seq[0])
    assert not batched[:, 2].any()                       # the -100 scene: zero rows
    assert batched[:, 0].any()
    if mode == 0 or e:                                   # mode 1 without contacts or equality rows: zhat = 0
        assert batched[:, 1].any()


@pytest.mark.parametrize("R", [1, 7, "n"])
@pytest.mark.parametrize("e", [0, 3])
@pytest.mark.parametrize("mode", [0, 1])
def test_forced_banded_batched_jvp_equals_sequential(forced_banded, mode, e, R):
    forced_banded(True)
    nb, nc = 16, 30
    ins, A, b, b1, b2, counts = _soa_case(5, nb, nc, e, f64, seed=21, special=True)
    R = 3 * nb if R == "n" else R
    batched, seq, dual, status = _batched_and_sequential_jvp(ins, A, b, b1, b2, counts, mode, R, seed=R)
    assert int(status[2]) == -100, status.tolist()
    assert not batched[:, 2].any()
    keep = [s for s in range(5) if s != 2]
    assert _row_scale_err(batched[:, keep], seq[:, keep]) <= 1e-10
    assert _row_scale_err(dual[None, keep], seq[0:1, keep]) <= 1e-10


def test_second_order_and_vmap_over_the_solve_raise():
    ins, A, b, b1, b2, counts = _soa_case(3, 4, 5, 0, f64, seed=1, special=False)
    f = _solve_fn(b1, b2, 0, True, counts, 0)
    v = ins[2]
    g = lambda x: f(*ins[:2], x, *ins[3:])
    with pytest.raises(NotImplementedError, match="vmap over the inputs"):
        torch.func.vmap(lambda x: torch.func.jvp(g, (x,), (torch.ones_like(x),))[1])(v.unsqueeze(0).expand(2, -1, -1))
    with pytest.raises(NotImplementedError, match="second derivatives"):
        torch.func.jvp(lambda x: torch.func.jvp(g, (x,), (torch.ones_like(x),))[1], (v,), (torch.ones_like(v),))
    with pytest.raises(NotImplementedError, match="second derivatives"):
        torch.func.vjp(lambda x: torch.func.jvp(g, (x,), (torch.ones_like(x),))[1], v)[1](torch.ones_like(v))


# ------------------------------------------------------------------ 4. a step
def _step_fn(w):
    """f(x, u) = the state after one step from x = (p, v) with the extra generalised force u, as linearize() runs it."""
    B, n = w.B, w.n
    ef = w.external_force

    def f(x, u):
        w.p = x[:, :n].reshape(B, w.nd, 3)
        w.v = x[:, n:]
        ub = u.reshape(B, w.nd, 3)
        w.external_force = (lambda t: ub) if ef is None else (lambda t: ef(t) + ub)
        w.find_contacts()
        w.step_dt(w.dt)
        return torch.cat([w.get_p(), w.v], 1)
    return f


def _restore(w, saved, joints):
    w.__dict__.clear()
    w.__dict__.update(saved)
    for st, old in zip(w._jstate, joints):
        if st is not None:
            st[:] = old


def _jacfwd_step(w):
    """Per-scene (A, Bu) of one step by jacfwd with one-hot tangents placed in every scene at once."""
    saved, joints = dict(w.__dict__), [None if st is None else list(st) for st in w._jstate]
    B, n = w.B, w.n
    x0 = torch.cat([w.get_p(), w.v], 1).detach()
    u0 = x0.new_zeros(B, n)
    f = _step_fn(w)
    try:
        eye = torch.eye(3 * n, dtype=x0.dtype, device=x0.device).unsqueeze(1).expand(-1, B, -1)
        J = torch.func.vmap(lambda t: torch.func.jvp(f, (x0, u0), (t[:, :2 * n], t[:, 2 * n:]))[1])(eye)
    finally:
        _restore(w, saved, joints)
    return J[:2 * n].permute(1, 2, 0), J[2 * n:].permute(1, 2, 0)          # [B, 2n, 2n], [B, 2n, n]


@pytest.mark.parametrize("scene", ["pile_bin", "polygon_bin", "chain", "pile60_banded"])
def test_jacfwd_of_a_step_equals_exact_linearize(scene):
    w = _scene(scene)
    w.exact_adjoint = True
    before = (w.p.clone(), w.v.clone(), w.t.clone())
    _, A, Bu = w.linearize()
    Af, Bf = _jacfwd_step(w)
    assert torch.equal(w.p, before[0]) and torch.equal(w.v, before[1]) and torch.equal(w.t, before[2])
    # resting piles and boxes: sticking contacts whose solves stall leave d = lam / s at the clamp, W ~ 1e10, and the
    # contact-geometry terms of the right-hand side pass through it; K and K^T solves then agree to ~1e-8
    tol = 1e-8 if scene in ("pile_bin", "polygon_bin") else 1e-10
    assert _rel(Af, A) <= tol and _rel(Bf, Bu) <= tol, (_rel(Af, A), _rel(Bf, Bu))


@pytest.mark.parametrize("scene", ["row8_rect_floor", "polygons_sliding"])
def test_step_jvp_through_contact_geometry_matches_finite_differences(scene):
    """The tangent along a random (dx, du) -- it moves polygon poses -- and, on the Rect floor, along the obstacle's
    vertices: non-zero and equal to central differences of plain steps with the same contact and dt-halving history.
    With the kernel's geometry these tangents would miss every contact-geometry term."""
    w = _sliding_balls(2, 8, seed=3, floor="rect") if scene == "row8_rect_floor" else _polygon_bin(2, slide=True)
    base = torch.cat([w.get_p(), w.v], 1).detach()
    gen = torch.Generator().manual_seed(11)
    dx = torch.randn(base.shape, generator=gen, dtype=f64).cuda()
    du = 100.0 * torch.randn(w.B, w.n, generator=gen, dtype=f64).cuda()
    saved, joints = dict(w.__dict__), [None if st is None else list(st) for st in w._jstate]
    try:
        _, an = torch.func.jvp(_step_fn(w), (base, base.new_zeros(w.B, w.n)), (dx, du))
    finally:
        _restore(w, saved, joints)
    _, hist = _step_from(w, base, base.new_zeros(w.B, w.n))
    h = 1e-6
    xp, hp = _step_from(w, base + h * dx, h * du)
    xm, hm = _step_from(w, base - h * dx, -h * du)
    assert hp == hist and hm == hist, (hist, hp, hm)
    fd = (xp - xm) / (2 * h)
    assert float(an.abs().max()) > 0
    err = float(((an - fd).abs().max(1)[0] / fd.abs().max(1)[0]).max())
    assert err < 1e-4, err
    if scene != "row8_rect_floor":
        return
    # the floor's vertices: a tangent that reaches the step only through the contact geometry
    from lcp_physics_b200.world import polygon_centroid
    ov0 = w.ov.detach().clone()
    dv = torch.randn(ov0.shape, generator=gen, dtype=f64).cuda()

    def g(ov):
        w.ov, w.oref = ov, polygon_centroid(ov)
        w.find_contacts()
        w.step()
        return torch.cat([w.get_p(), w.v], 1)

    try:
        _, an = torch.func.jvp(g, (ov0,), (dv,))
    finally:
        _restore(w, saved, joints)
    outs = []
    for s in (1, -1):
        try:
            with torch.no_grad():
                outs.append(g(ov0 + s * h * dv))
        finally:
            _restore(w, saved, joints)
    fd = (outs[0] - outs[1]) / (2 * h)
    assert float(an.abs().max()) > 1e-3 * float(fd.abs().max()) > 0
    err = float(((an - fd).abs().max(1)[0] / fd.abs().max(1)[0]).max())
    assert err < 1e-4, err


# ------------------------------------------------------------------ 5. a rollout
def _rollout_world(scene, theta):
    """The world with theta = (friction offset, relative mass change, initial velocity change along a fixed
    direction) applied to the parameters it is built from."""
    from lcp_physics_b200.scenes import make_ball_pile
    from lcp_physics_b200.world import BatchedWorld, Joint, XConstraint, YConstraint, rect_vertices
    if scene == "sliding":
        B, nballs, R, r = 2, 8, 1.0e5, 10.0
        ic = make_ball_pile(B, nballs=nballs, cols=nballs, seed=3, gap=30.0, r=r, r_floor=R)
        gen = torch.Generator().manual_seed(3)
        rnd = lambda: torch.rand(B, nballs, generator=gen, dtype=f64)
        # sliding for the whole rollout: no ball stops or catches up with the next one
        ic["vel"][:, 1:, 1] = 48.0 + 4.0 * rnd()
        ic["vel"][:, 1:, 2] = 1.5
        ic["vel"][:, 1:, 0] = rnd() - 0.5
        ic["fric"][:, 1:] = 0.05 + 0.1 * rnd()
        ic["rest"][:, 1:] = 0.2 + 0.5 * rnd()
        ic["pos"][:, 1:, 1] = 500.0 - r - 0.05
        x = ic["pos"][0, 1:, 0]
        lo, hi = float(x.min()) - 100.0, float(x.max()) + 1200.0
        floor_v = rect_vertices([0.5 * (lo + hi), 510.0], [hi - lo, 20.0]).unsqueeze(0)
        dv = torch.zeros(B, nballs, 3, dtype=f64)
        dv[..., 1] = 1.0
        vel = ic["vel"][:, 1:].cuda() + theta[2] * dv.cuda()
        return BatchedWorld(ic["pos"][:, 1:], ic["rad"][:, 1:], vel=vel, mass=ic["mass"][:, 1:].cuda() * (1 + theta[1]),
                            restitution=ic["rest"][:, 1:], fric_coeff=ic["fric"][:, 1:].cuda() + theta[0],
                            obstacles=floor_v, obstacle_fric=0.3, obstacle_rest=0.4, gravity=100.0, dt=DT,
                            max_iter=40, exact_adjoint=True, device="cuda")
    B = 2
    g = torch.Generator().manual_seed(0)
    links = torch.stack([rect_vertices([300.0, 50.0 + 50.0 * i], [20.0, 60.0]) for i in range(10)])
    cons = [XConstraint(1), YConstraint(1)] + [Joint(1 + i, i, [300.0, 25.0 + 50.0 * i]) for i in range(1, 10)]
    pos = torch.stack([torch.full((B,), 200.0, dtype=f64), 500.0 + 20.0 * (torch.rand(B, generator=g, dtype=f64) - 0.5)],
                      1).unsqueeze(1)
    vel = torch.zeros(B, 1, 3, dtype=f64, device="cuda")
    vel = vel + theta[2] * torch.tensor([0.0, 1.0, 0.0], dtype=f64, device="cuda")

    def push(t):
        f = torch.zeros(B, 11, 3, dtype=t.dtype, device=t.device)
        f[:, 0, 1] = torch.where(t < 0.1, torch.full_like(t, 2000.0), torch.zeros_like(t))
        return f
    return BatchedWorld(pos, 20.0, vel=vel, mass=1.0 + theta[1], fric_coeff=0.9 + theta[0], restitution=0.9,
                        gravity=100.0, gravity_mask=[False, False] + [True] * 9, dt=DT, post_stab=True,
                        polygons=links.unsqueeze(0).expand(B, -1, -1, -1), poly_rest=0.9, constraints=cons,
                        no_contact=[(1 + i, i) for i in range(1, 10)], external_force=push, exact_adjoint=True,
                        max_iter=40, device="cuda")


def _rollout(scene, T):
    def f(theta):
        w = _rollout_world(scene, theta)
        hist = []
        for _ in range(T):
            w.step()
            hist.append((w.counts.tolist(), w.t.tolist()))
        f.hist = hist
        return torch.cat([w.get_p(), w.v], 1)
    return f


@pytest.mark.parametrize("scene", ["sliding", "chain"])
def test_rollout_sensitivities_forward_equals_reverse_and_finite_differences(scene):
    T = 30
    f = _rollout(scene, T)
    theta = torch.zeros(3, dtype=f64, device="cuda")
    Jf = torch.func.jacfwd(f, randomness="same")(theta)      # the scene builders draw random numbers
    Jr = torch.func.jacrev(f)(theta)
    assert Jf.shape == (2, 2 * _rollout_world(scene, theta).n, 3)
    assert float(Jf.abs().max()) > 0
    # relative to the whole Jacobian: a parameter the rollout barely depends on (the chain's friction) has a
    # column at round-off level
    rel = float((Jf - Jr).norm() / Jr.norm())
    assert rel <= 1e-4, rel
    with torch.no_grad():
        f(theta)
        hist = f.hist
        h = 1e-6
        checked = []
        for k in range(3):
            d = torch.zeros(3, dtype=f64, device="cuda")
            d[k] = h
            xp = f(theta + d)
            hp = f.hist
            xm = f(theta - d)
            if scene == "chain" and not (hp == hist and f.hist == hist):
                # the projectile's impact ends a step at the penetration tolerance: a lighter projectile takes one more
                # dt halving there, and the quotient then spans two branches of the rollout -- not a derivative
                continue
            assert hp == hist and f.hist == hist, k
            fd = (xp - xm) / (2 * h)
            err = float((Jf[..., k] - fd).abs().max() / Jf.abs().max())
            assert err < 1e-4, (k, err)
            checked.append(k)
        assert len(checked) >= (3 if scene == "sliding" else 2), checked


def test_forward_mode_rollout_memory_does_not_grow_with_length():
    theta = torch.zeros(3, dtype=f64, device="cuda")
    peaks = {}
    for T in (10, 40):
        f = _rollout("sliding", T)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        torch.func.jacfwd(f, randomness="same")(theta)
        torch.cuda.synchronize()
        peaks[T] = torch.cuda.max_memory_allocated() - base
    assert peaks[40] <= 1.1 * peaks[10], peaks
