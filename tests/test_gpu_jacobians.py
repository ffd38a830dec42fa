"""GPU: Jacobians through the engine solve and `BatchedWorld.linearize`.

1. `torch.func.vmap` of an `engine_solve` vector-Jacobian product (one lcpb200_engine_backward_batched call with R
   cotangents) equals R separate calls of the existing backward: bitwise on the condensed kernels, within the banded
   kernel's atomic-order noise; a scene with status -100 gets zero rows and leaves the others alone; the result does
   not depend on how the kernel chunks the cotangents of a scene.
2. `torch.func.jacrev` of `engine_solve` against central differences on converged solves (exact adjoint).
3. `BatchedWorld.linearize` against R row-by-row `torch.autograd.grad` calls through a normal step, and against
   central differences of `step()` on scenes whose solves converge; fp32 against fp64.
4. `linearize` leaves the world as it was, and its x_next is the state `step()` reaches.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
NAMES = ["mass", "inertia", "v", "fext", "normal", "p1", "p2", "mu", "restitution"]
DT = 1.0 / 30
f64 = torch.float64


@pytest.fixture
def forced_banded():
    import os

    from lcp_physics_b200 import _lib

    def set_(on):
        if on:
            os.environ["LCPB200_FORCE_BANDED"] = "1"
        else:
            os.environ.pop("LCPB200_FORCE_BANDED", None)
        _lib.clear_handles()
    yield set_
    set_(False)


# ------------------------------------------------------------------ engine_solve scenes
def _soa_case(B, nb, nc, e, dtype, seed, special):
    """Random contact lists (make_contact_soa) with per-scene counts; special: scene 1 has no contact and scene 2 a
    contact of a body with itself (status -100)."""
    from lcp_physics_b200.scenes import make_contact_soa
    soa = dict(make_contact_soa(B, nb, nc, seed=seed))
    fext = torch.zeros(B, 3 * nb, dtype=f64)
    fext[:, 2::3] = 10.0 * soa["mass"]
    soa["fext"] = fext
    b1 = soa["body1"].unsqueeze(0).expand(B, -1).contiguous()
    b2 = soa["body2"].unsqueeze(0).expand(B, -1).contiguous()
    counts = torch.full((B,), nc, dtype=torch.int32)
    if special:
        counts[1] = 0
        b2[2, 0] = b1[2, 0]
    ins = [soa[k].to(dtype).cuda() for k in NAMES]
    A = b = None
    if e:
        A = torch.zeros(B, e, 3 * nb, dtype=dtype)
        A[:, torch.arange(e), torch.arange(e)] = 1
        A, b = A.cuda(), torch.zeros(B, e, dtype=dtype).cuda()
    return ins, A, b, b1.cuda(), b2.cuda(), counts.cuda()


def _solve_fn(b1, b2, mode, exact, counts, e, max_iter=10):
    from lcp_physics_b200.engines import engine_solve

    def f(*x):
        return engine_solve(*x[:9], b1, b2, DT, A=x[9] if e else None, b=x[10] if e else None, mode=mode,
                            max_iter=max_iter, exact_adjoint=exact, counts=counts)[0]
    return f


def _batched_and_sequential(ins, A, b, b1, b2, counts, mode, exact, R, seed):
    """vmap(vjp_fn)(G) and R torch.autograd.grad calls (the existing backward) for the same cotangents G [R, B, n]."""
    e = 0 if A is None else A.shape[1]
    f = _solve_fn(b1, b2, mode, exact, counts, e)
    args = ins + ([A, b] if e else [])
    z, vjp_fn = torch.func.vjp(f, *args)
    B, n = z.shape
    gen = torch.Generator().manual_seed(seed)
    G = torch.randn(R, B, n, generator=gen, dtype=f64).to(z.dtype).cuda()
    batched = torch.func.vmap(vjp_fn)(G)
    leaves = [t.clone().requires_grad_(True) for t in args]
    zz = f(*leaves)
    seq = [torch.autograd.grad(zz, leaves, G[r], retain_graph=True) for r in range(R)]
    seq = [torch.stack([s[i] for s in seq]) for i in range(len(args))]
    from lcp_physics_b200.engines import last_solve_info
    return batched, seq, last_solve_info()["status"]


@pytest.mark.parametrize("B", [4, 300])                 # 4: several chunks of cotangents per scene; 300: one
@pytest.mark.parametrize("R", [1, 7, "n"])
@pytest.mark.parametrize("e", [0, 3])
@pytest.mark.parametrize("exact", [False, True])
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_condensed_batched_vjp_equals_sequential_backward(dtype, mode, exact, e, R, B):
    nb, nc = 6, 8
    ins, A, b, b1, b2, counts = _soa_case(B, nb, nc, e, dtype, seed=3, special=True)
    R = 3 * nb if R == "n" else R
    batched, seq, status = _batched_and_sequential(ins, A, b, b1, b2, counts, mode, exact, R, seed=R + B)
    assert int(status[2]) == -100 and int(status[1]) >= 0, status.tolist()
    for name, x, y in zip(NAMES + ["A", "b"], batched, seq):
        assert x.shape == y.shape, name
        assert torch.equal(x, y), (name, float((x - y).abs().max()))
        assert not x[:, 2].any(), name                       # the -100 scene: zero rows
    assert any(bool(x[:, 0].any()) for x in batched)


def _row_scale_err(x, y):
    """max over cotangents r of |x_r - y_r| / max |y_r|, the error relative to each row's scale."""
    x, y = x.reshape(x.shape[0], -1).double(), y.reshape(y.shape[0], -1).double()
    return float(((x - y).abs().max(1)[0] / y.abs().max(1)[0].clamp_min(1e-300)).max())


@pytest.mark.parametrize("R", [1, 7, "n"])
@pytest.mark.parametrize("e", [0, 3])
@pytest.mark.parametrize("exact", [False, True])
@pytest.mark.parametrize("mode", [0, 1])
def test_forced_banded_batched_vjp_equals_sequential_backward(forced_banded, mode, exact, e, R):
    forced_banded(True)
    nb, nc = 16, 30
    ins, A, b, b1, b2, counts = _soa_case(5, nb, nc, e, f64, seed=21, special=True)
    R = 3 * nb if R == "n" else R
    batched, seq, status = _batched_and_sequential(ins, A, b, b1, b2, counts, mode, exact, R, seed=R)
    assert int(status[2]) == -100, status.tolist()
    for name, x, y in zip(NAMES + ["A", "b"], batched, seq):
        assert not x[:, 2].any(), name
        keep = [s for s in range(5) if s != 2]
        if bool(y[:, keep].any()):
            # fp64 atomics in the banded assembly: the sum order differs from call to call
            assert _row_scale_err(x[:, keep], y[:, keep]) <= 1e-10, name


def _sliding_balls(B, nballs, seed, dtype=f64, floor="ball"):
    """`nballs` balls (radius 10, 10 apart: they touch only the floor) on the floor, sliding the same way at 40 .. 60,
    spinning and moving towards the floor, friction 0.1 .. 0.4: every contact slides for the whole step, so every
    solve converges far below 1e-8 and the step is a smooth map of the state. floor "ball": a pinned floor ball of
    radius 1e5 (body 0); "rect": a Rect obstacle floor whose top is y = 500."""
    from lcp_physics_b200.scenes import make_ball_pile
    R, r = 1.0e5, 10.0
    ic = make_ball_pile(B, nballs=nballs, cols=nballs, seed=seed, gap=10.0, r=r, r_floor=R)
    dx = ic["pos"][:, 1:, 0] - 500.0
    ic["pos"][:, 1:, 1] = 500.0 + R - torch.sqrt((R + r + 0.05) ** 2 - dx * dx)
    gen = torch.Generator().manual_seed(seed)
    rnd = lambda: torch.rand(B, nballs, generator=gen, dtype=f64)
    ic["vel"][:, 1:, 1] = 40.0 + 20.0 * rnd()
    ic["vel"][:, 1:, 2] = 1.5
    ic["vel"][:, 1:, 0] = rnd() - 0.5
    ic["fric"][:, 1:] = 0.1 + 0.3 * rnd()
    ic["rest"][:, 1:] = 0.2 + 0.5 * rnd()
    ic = {k: v.to(dtype) for k, v in ic.items()}
    from lcp_physics_b200.world import BatchedWorld, rect_vertices
    kw = dict(gravity=100.0, dt=DT, max_iter=40, exact_adjoint=True, device="cuda")
    if floor == "ball":
        return BatchedWorld(ic["pos"], ic["rad"], vel=ic["vel"], mass=ic["mass"], restitution=ic["rest"],
                            fric_coeff=ic["fric"], static=[0], **kw)
    ic["pos"][:, 1:, 1] = 500.0 - r - 0.05
    x = ic["pos"][0, 1:, 0]
    lo, hi = float(x.min()) - 100.0, float(x.max()) + 400.0
    floor_v = rect_vertices([0.5 * (lo + hi), 510.0], [hi - lo, 20.0]).to(dtype).unsqueeze(0)
    return BatchedWorld(ic["pos"][:, 1:], ic["rad"][:, 1:], vel=ic["vel"][:, 1:], mass=ic["mass"][:, 1:],
                        restitution=ic["rest"][:, 1:], fric_coeff=ic["fric"][:, 1:], obstacles=floor_v,
                        obstacle_fric=0.3, obstacle_rest=0.4, **kw)


def _world_soa(w):
    soa = dict(mass=w.mass, inertia=w.inertia, v=w.v, fext=w.fext, normal=w.c_normal, p1=w.c_p1, p2=w.c_p2,
               mu=w.c_mu, restitution=w.c_rest)
    return [soa[k].detach().clone() for k in NAMES]


def test_natural_banded_batched_vjp_equals_sequential_backward():
    """A 46-body world (n + e > 128): the banded kernel by itself, per-scene counts, a pinned floor in the border."""
    w = _sliding_balls(1, 45, seed=3)
    assert w.large
    ins = _world_soa(w)
    b = torch.zeros(1, w.ne, dtype=f64, device="cuda")
    for R in (1, 7, w.n):
        batched, seq, status = _batched_and_sequential(ins, w.A, b, w.c_b1, w.c_b2, w.counts, 0, True, R, seed=R)
        assert (status >= 0).all()
        for name, x, y in zip(NAMES + ["A", "b"], batched, seq):
            if bool(y.any()):
                assert _row_scale_err(x, y) <= 1e-10, (R, name)


def test_vmap_over_the_solve_raises():
    ins, A, b, b1, b2, counts = _soa_case(3, 4, 5, 0, f64, seed=1, special=False)
    f = _solve_fn(b1, b2, 0, True, counts, 0)
    with pytest.raises(NotImplementedError, match="vmap over the inputs"):
        torch.func.vmap(lambda v: f(*ins[:2], v, *ins[3:]))(ins[2].unsqueeze(0).expand(2, -1, -1))


# ------------------------------------------------------------------ 2. jacrev against finite differences
@pytest.mark.parametrize("scene", ["row8_condensed", "row8_forced_banded", "row45_banded"])
def test_jacrev_matches_finite_differences(forced_banded, scene):
    """Jacobians of zhat of one converged solve (status >= 0, residual < 1e-8, exact adjoint) w.r.t. v, fext, normal,
    p1, p2, mu and the equality rows A (the floor ball's pin), from torch.func.jacrev, against central differences
    along random directions."""
    from lcp_physics_b200.engines import last_solve_info
    forced_banded(scene == "row8_forced_banded")
    w = _sliding_balls(1, 45 if scene == "row45_banded" else 8, seed=3)
    assert w.large == (scene == "row45_banded")
    ins = _world_soa(w)
    A, b = w.A.detach().clone(), torch.zeros(1, w.ne, dtype=f64, device="cuda")
    f = _solve_fn(w.c_b1, w.c_b2, 0, True, w.counts, w.ne, max_iter=40)
    args = ins + [A, b]
    f(*args)
    st, resid = last_solve_info()["status"], last_solve_info()["resid"]
    assert (st >= 0).all() and float(resid.max()) < 1e-8, (st.tolist(), resid.tolist())
    which = {"v": 2, "fext": 3, "normal": 4, "p1": 5, "p2": 6, "mu": 7, "A": 9}
    jac = torch.func.jacrev(f, argnums=tuple(which.values()))(*args)
    gen = torch.Generator().manual_seed(7)
    h = 1e-6
    worst, scale = {}, {}
    for (name, i), J in zip(which.items(), jac):
        d = torch.randn(args[i].shape, generator=gen, dtype=f64).cuda()
        if name == "normal":
            d = d - (d * args[i]).sum(-1, keepdim=True) * args[i]              # stay on the unit circle to first order
        if name == "A":
            # within the rows' pattern (the pinned body's columns): the large-scene kernel takes its border from it
            d = d * (args[i] != 0).any(1, keepdim=True)
        plus = [t + h * d if j == i else t for j, t in enumerate(args)]
        minus = [t - h * d if j == i else t for j, t in enumerate(args)]
        fd = (f(*plus) - f(*minus)) / (2 * h)
        an = (J * d.reshape((1, 1) + tuple(d.shape))).flatten(2).sum(2)
        worst[name], scale[name] = float((an - fd).abs().max()), float(fd.abs().max())
    top = max(scale.values())
    # p1 is the contact point on body 1, here the pinned floor ball: zhat does not depend on it (both sides ~1e-10)
    rel = {k: worst[k] / (scale[k] if scale[k] > 1e-6 * top else top) for k in worst}
    assert max(rel.values()) < 1e-4, sorted(rel.items(), key=lambda kv: -kv[1])


# ------------------------------------------------------------------ 3. / 4. BatchedWorld.linearize
def _pile_bin(B, dtype=f64):
    """24-ball piles (6 wide, 0.05 apart) in a bin of three Rect obstacles: floor and two walls."""
    from lcp_physics_b200.scenes import make_ball_pile
    from lcp_physics_b200.world import BatchedWorld, rect_vertices
    ic = make_ball_pile(B, nballs=24, cols=6, seed=2000, gap=0.05)
    x = ic["pos"][0, 1:, 0]
    lo, hi = float(x.min()) - 10.0, float(x.max()) + 10.0
    obst = torch.stack([rect_vertices([0.5 * (lo + hi), 510.0], [hi - lo + 200.0, 20.0]),
                        rect_vertices([lo - 11.0, 300.0], [20.0, 398.0]), rect_vertices([hi + 11.0, 300.0], [20.0, 398.0])])
    return BatchedWorld(ic["pos"][:, 1:].to(dtype), ic["rad"][:, 1:].to(dtype), vel=ic["vel"][:, 1:].to(dtype),
                        mass=ic["mass"][:, 1:], restitution=ic["rest"][:, 1:], fric_coeff=ic["fric"][:, 1:],
                        gravity=100.0, dt=DT, obstacles=obst.to(dtype), obstacle_fric=0.9, obstacle_rest=0.5,
                        device="cuda")


def _polygon_bin(B, slide=False):
    """3 boxes and a hexagon on the floor of a bin, 4 circles on top of them; slide: the boxes and the hexagon slide
    along the floor (every contact slides) and nothing rests on them."""
    from lcp_physics_b200.world import BatchedWorld, rect_vertices
    g = torch.Generator().manual_seed(5)
    tilt = 0.1 if slide else 0.0           # tilted: one corner on the floor, no tie between reference faces
    polys = []
    for k in range(4):
        cx = 100.0 + 40.0 * k
        if k == 3:
            t = torch.arange(6, dtype=f64) * (math.pi / 3) + tilt
            v = torch.stack([cx + 9.0 * torch.cos(t), 9.0 * torch.sin(t)], 1)
        else:
            v = rect_vertices([cx, 0.0], [30.0, 16.0], tilt)
            v = torch.cat([v, v[3:].expand(2, 2)])
        v[:, 1] += 500.0 - 0.03 - v[:, 1].max()                             # lowest vertex 0.03 above the floor
        polys.append(v)
    pv = torch.stack(polys).unsqueeze(0).repeat(B, 1, 1, 1)
    pv[..., 0] += 0.5 * (torch.rand(B, 4, 1, generator=g, dtype=f64) - 0.5)
    obst = torch.stack([rect_vertices([300.0, 510.0], [1000.0, 20.0]), rect_vertices([60.0, 400.0], [20.0, 220.0]),
                        rect_vertices([760.0, 400.0], [20.0, 220.0])])
    obst = torch.cat([obst, obst[:, 3:].expand(-1, 2, -1)], 1)
    if slide:
        pvel = torch.zeros(B, 4, 3, dtype=f64)
        pvel[..., 1] = 30.0 + 20.0 * torch.rand(B, 4, generator=g, dtype=f64)
        pvel[..., 2] = 1.0
        pos = torch.tensor([[[400.0, 300.0]]], dtype=f64).expand(B, 1, 2)
        return BatchedWorld(pos, 6.0, gravity=100.0, dt=DT, polygons=pv, obstacles=obst, poly_vel=pvel,
                            obstacle_fric=0.3, obstacle_rest=0.3, poly_fric=0.3, poly_rest=0.3, max_iter=40,
                            exact_adjoint=True, device="cuda")
    pos = torch.stack([100.0 + 40.0 * torch.arange(4, dtype=f64).expand(B, -1) + torch.rand(B, 4, generator=g, dtype=f64),
                       torch.full((B, 4), 500.0 - 16.03 - 6.0 - 0.03, dtype=f64)], 2)
    return BatchedWorld(pos, 6.0, gravity=100.0, dt=DT, polygons=pv, obstacles=obst, obstacle_fric=0.6,
                        obstacle_rest=0.3, poly_fric=0.5, poly_rest=0.3, fric_coeff=0.5, restitution=0.3, device="cuda")


def _chain(B, dtype=f64, exact=False):
    """chain_demo: 10 Rect links (X and Y constraints on the top link, 9 Joints, no_contact between neighbours),
    Gravity on the links, a projectile circle pushed towards the chain for t < 0.1, post-stabilisation."""
    from lcp_physics_b200.world import BatchedWorld, Joint, XConstraint, YConstraint, rect_vertices
    g = torch.Generator().manual_seed(0)
    links = torch.stack([rect_vertices([300.0, 50.0 + 50.0 * i], [20.0, 60.0]) for i in range(10)])
    cons = [XConstraint(1), YConstraint(1)] + [Joint(1 + i, i, [300.0, 25.0 + 50.0 * i]) for i in range(1, 10)]
    pos = torch.stack([torch.full((B,), 200.0, dtype=f64), 500.0 + 20.0 * (torch.rand(B, generator=g, dtype=f64) - 0.5)],
                      1).unsqueeze(1)

    def push(t):
        f = torch.zeros(B, 11, 3, dtype=t.dtype, device=t.device)
        f[:, 0, 1] = torch.where(t < 0.1, torch.full_like(t, 2000.0), torch.zeros_like(t))
        return f
    return BatchedWorld(pos.to(dtype), 20.0, restitution=0.9, gravity=100.0, gravity_mask=[False, False] + [True] * 9,
                        dt=DT, post_stab=True, polygons=links.unsqueeze(0).expand(B, -1, -1, -1).to(dtype),
                        poly_rest=0.9, constraints=cons, no_contact=[(1 + i, i) for i in range(1, 10)],
                        external_force=push, exact_adjoint=exact, max_iter=40, device="cuda")


def _pile60():
    """One 60-ball pile on a pinned floor ball: n = 183 > 128, the banded kernel."""
    from lcp_physics_b200.scenes import make_ball_pile
    from lcp_physics_b200.world import BatchedWorld
    ic = make_ball_pile(1, nballs=60, cols=12, seed=4, gap=0.05)
    return BatchedWorld(ic["pos"], ic["rad"], vel=ic["vel"], mass=ic["mass"], restitution=ic["rest"],
                        fric_coeff=ic["fric"], gravity=100.0, static=[0], dt=DT, device="cuda")


def _scene(name):
    if name == "pile_bin":
        return _pile_bin(2)
    if name == "polygon_bin":
        return _polygon_bin(2)
    if name == "chain":
        w = _chain(2)
        for _ in range(12):                                   # the chain swinging, the projectile flying towards it
            w.step()
        return w
    w = _pile60()
    w.step()
    return w


def _state(w):
    """Everything a step reads or writes: state, joint state, contact list."""
    keys = ["p", "v", "t", "A", "counts", "c_b1", "c_b2", "c_normal", "c_p1", "c_p2", "c_pen", "c_mu", "c_rest"]
    out = {k: getattr(w, k) for k in keys if getattr(w, k, None) is not None}
    out["joints"] = [None if st is None else list(st) for st in w._jstate]
    return out


def _same_state(a, b):
    assert a.keys() == b.keys()
    for k in a:
        if k == "joints":
            for sa, sb in zip(a[k], b[k]):
                assert (sa is None) == (sb is None)
                if sa is not None:
                    assert all(torch.equal(x, y) for x, y in zip(sa, sb)), k
        else:
            assert torch.equal(a[k], b[k]), k


def _step_from(w, x, u):
    """x_next = f(x, u) by a plain step() from state x with the extra generalised force u (no autograd); also the
    contact counts at x and after the step and the step's times (its dt-halving history). The world is restored."""
    saved = dict(w.__dict__)
    joints = [None if st is None else list(st) for st in w._jstate]
    ef, n = w.external_force, w.n
    try:
        with torch.no_grad():
            w.p = x[:, :n].reshape(w.B, w.nd, 3).clone()
            w.v = x[:, n:].clone()
            ub = u.reshape(w.B, w.nd, 3)
            w.external_force = (lambda t: ub) if ef is None else (lambda t: ef(t) + ub)
            w.find_contacts()
            feat = lambda: [f[:c] for f, c in zip(w.c_feat.tolist(), w.counts.tolist())] if w.np else None
            c0, f0 = w.counts.tolist(), feat()
            w.step()
            return torch.cat([w.get_p(), w.v], 1), (c0, f0, w.counts.tolist(), feat(), (w.t - saved["t"]).tolist())
    finally:
        w.__dict__.clear()
        w.__dict__.update(saved)
        for st, old in zip(w._jstate, joints):
            if st is not None:
                st[:] = old


def _rows_autograd(w):
    """The Jacobian rows of a normal step, one torch.autograd.grad call per output row."""
    saved = dict(w.__dict__)
    joints = [None if st is None else list(st) for st in w._jstate]
    ef, n, B = w.external_force, w.n, w.B
    try:
        x = torch.cat([w.get_p(), w.v], 1).detach().clone().requires_grad_(True)
        u = x.new_zeros(B, n).requires_grad_(True)
        w.p = x[:, :n].reshape(B, w.nd, 3)
        w.v = x[:, n:]
        ub = u.reshape(B, w.nd, 3)
        w.external_force = (lambda t: ub) if ef is None else (lambda t: ef(t) + ub)
        w.find_contacts()
        w.step()
        out = torch.cat([w.get_p(), w.v], 1)
        rows = [torch.autograd.grad(out[:, r].sum(), (x, u), retain_graph=True) for r in range(2 * n)]
        return torch.stack([r[0] for r in rows], 1), torch.stack([r[1] for r in rows], 1)
    finally:
        w.__dict__.clear()
        w.__dict__.update(saved)
        for st, old in zip(w._jstate, joints):
            if st is not None:
                st[:] = old


def _rel(a, b):
    a, b = a.reshape(a.shape[0], -1), b.reshape(b.shape[0], -1)
    return float(((a - b).norm(dim=1) / b.norm(dim=1).clamp_min(1e-300)).max())


@pytest.mark.parametrize("scene", ["pile_bin", "polygon_bin", "chain", "pile60_banded"])
def test_linearize_matches_autograd_rows_and_leaves_the_world_unchanged(scene):
    w = _scene(scene)
    assert w.large == (scene == "pile60_banded")
    before = _state(w)
    x_next, A, Bu = w.linearize()
    _same_state(before, _state(w))
    n = w.n
    assert A.shape == (w.B, 2 * n, 2 * n) and Bu.shape == (w.B, 2 * n, n)
    assert torch.isfinite(A).all() and torch.isfinite(Bu).all()
    Ar, Br = _rows_autograd(w)
    _same_state(before, _state(w))
    assert _rel(A, Ar) <= 1e-12 and _rel(Bu, Br) <= 1e-12, (_rel(A, Ar), _rel(Bu, Br))
    twin = _scene(scene)                                      # a world that never linearised
    w.step()
    twin.step()
    assert torch.equal(w.p, twin.p) and torch.equal(w.v, twin.v) and torch.equal(w.t, twin.t)
    ref = torch.cat([before["p"].reshape(w.B, n), before["v"]], 1)
    step_x = torch.cat([w.get_p(), w.v], 1)
    assert _rel(x_next, step_x) <= 1e-12, _rel(x_next, step_x)
    assert not torch.equal(ref, step_x)


@pytest.mark.parametrize("scene", ["pile_bin", "pile60_banded"])
def test_linearize_does_not_depend_on_chunk_size(scene):
    """Up to summation order: the backward of the torch geometry (gather -> scatter-add) accumulates with atomics, so
    two linearisations agree to round-off, not bit for bit; the kernel's own part is bitwise independent of its
    chunking (test_condensed_batched_vjp_equals_sequential_backward)."""
    w = _scene(scene)
    x0, A0, B0 = w.linearize()
    x1, A1, B1 = w.linearize(chunk_size=5)
    assert torch.equal(x0, x1)
    assert _rel(A1, A0) <= 1e-12 and _rel(B1, B0) <= 1e-12, (_rel(A1, A0), _rel(B1, B0))


def _fd_scene(name):
    if name == "row8_rect_floor":
        return _sliding_balls(2, 8, seed=3, floor="rect")
    if name == "polygons_sliding":
        return _polygon_bin(2, slide=True)
    if name == "chain":
        return _chain(2, exact=True)
    return _sliding_balls(1, 60, seed=3)


@pytest.mark.parametrize("scene", ["row8_rect_floor", "polygons_sliding", "chain", "row60_banded"])
def test_linearize_matches_finite_differences_of_step(scene):
    """A dx + Bu du against (f(x + h dx, h du) - f(x - h dx, -h du)) / 2h of plain step() calls, on scenes whose solves
    converge (sliding contacts, or equality rows only): with the same contact counts and dt halving on both sides the
    quotient is a derivative of the branch linearize describes."""
    from lcp_physics_b200.engines import last_solve_info
    w = _fd_scene(scene)
    assert w.large == (scene == "row60_banded")
    x0, A, Bu = w.linearize()
    if scene != "chain":                                      # the chain's solves have equality rows only
        assert float(last_solve_info()["resid"].max()) < 1e-8, last_solve_info()["resid"].tolist()
    base = torch.cat([w.get_p(), w.v], 1)
    _, hist = _step_from(w, base, base.new_zeros(w.B, w.n))
    gen = torch.Generator().manual_seed(11)
    dx = torch.randn(base.shape, generator=gen, dtype=f64).cuda()
    du = 100.0 * torch.randn(w.B, w.n, generator=gen, dtype=f64).cuda()
    h = 1e-6
    xp, hp = _step_from(w, base + h * dx, h * du)
    xm, hm = _step_from(w, base - h * dx, -h * du)
    assert hp == hist and hm == hist, (hist, hp, hm)
    fd = (xp - xm) / (2 * h)
    an = torch.bmm(A, dx.unsqueeze(2)).squeeze(2) + torch.bmm(Bu, du.unsqueeze(2)).squeeze(2)
    err = float(((an - fd).abs().max(1)[0] / fd.abs().max(1)[0]).max())
    assert err < 1e-4, err


def test_linearize_fp32_matches_fp64():
    """Sliding balls on a Rect floor in fp32 (condensed kernels) against the fp64 twin, each Jacobian relative to its
    norm."""
    w64, w32 = _sliding_balls(2, 8, seed=3, floor="rect"), _sliding_balls(2, 8, seed=3, dtype=torch.float32, floor="rect")
    _, A64, B64 = w64.linearize()
    _, A32, B32 = w32.linearize()
    assert A32.dtype == torch.float32
    assert _rel(A32.double(), A64) < 1e-3 and _rel(B32.double(), B64) < 1e-3, (_rel(A32.double(), A64),
                                                                                 _rel(B32.double(), B64))
