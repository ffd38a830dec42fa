"""GPU: ray casts against BatchedWorld scenes -- lcpb200_raycast, BatchedWorld.raycast and BatchedWorld.lidar.

* the kernel against the brute-force reference tests/ray_ref.py on seeded scenes (circles only; circles and obstacles;
  circles, padded polygons and obstacles; 256-vertex polygons; a world of thousands of bodies with `active`), fp32 and
  fp64, B in {1, 300}, R over several CTAs: body and feat equal, t to 1e-12 (fp64) / 1e-4 (fp32), the normal to
  1e-10 / 1e-3;
* determinism: two calls, and the same rays cast in a different split, are bitwise equal;
* per-scene activity: each scene reads what the standalone world of its active bodies reads;
* the torch mirror (graph path) equals the kernel path, and its gradients and tangents match central differences,
  jacrev matches jacfwd, and lidar readings after a 20-step rollout differentiate in both modes;
* lidar turns with its body; the entry point rejects bad arguments.
"""
import math

import pytest
import torch

from tests.ray_ref import ray_ref

pytestmark = pytest.mark.gpu
f64 = torch.float64


def hulls(g, B, n, V, L, sign=1.0, pad=True):
    """n random convex polygons per scene (vertices on a circle at sorted angles, 3..V of them), padded to V by
    repeating the last vertex (pad=False: V vertices each); sign -1 reverses every other polygon's orientation"""
    out = torch.empty(B, n, V, 2, dtype=f64)
    for s in range(B):
        for q in range(n):
            k = int(torch.randint(3, V + 1, (1,), generator=g)) if pad else V
            ang = torch.sort(torch.rand(k, generator=g, dtype=f64) * 2 * math.pi).values
            rr = 3 + 7 * float(torch.rand(1, generator=g))
            c = L * torch.rand(2, generator=g, dtype=f64)
            v = c + rr * torch.stack([torch.cos(ang), torch.sin(ang)], 1)
            if sign < 0 and q % 2:
                v = v.flip(0)
            out[s, q, :k] = v
            out[s, q, k:] = v[-1]
    return out


def scene(B, nb, np_, no, V, R, seed, L=100.0, pad=True):
    g = torch.Generator().manual_seed(seed)
    pos = L * torch.rand(B, nb, 2, generator=g, dtype=f64)
    rad = 1 + 4 * torch.rand(B, nb, generator=g, dtype=f64)
    pv = hulls(g, B, np_, V, L, pad=pad) if np_ else None
    ov = hulls(g, B, no, V, L, sign=-1.0, pad=pad) if no else None
    o = L * torch.rand(B, R, 2, generator=g, dtype=f64)
    a = 2 * math.pi * torch.rand(B, R, generator=g, dtype=f64)
    u = torch.stack([torch.cos(a), torch.sin(a)], 2)
    return dict(pos=pos, rad=rad, pv=pv, ov=ov, o=o, u=u)


def raw(sc, dtype, max_dist, active=None, normal=True):
    """lcpb200_raycast on the scene's tensors (cast to dtype): (t, body, feat, normal) on the GPU"""
    from lcp_physics_b200 import _lib
    from lcp_physics_b200.world import pack_bits
    lib = _lib.load()
    dv = lambda k: None if sc[k] is None else sc[k].to("cuda", dtype).contiguous()
    pos, rad, pv, ov, o, u = (dv(k) for k in ("pos", "rad", "pv", "ov", "o", "u"))
    B, R = o.shape[:2]
    nv = (pv if pv is not None else ov).shape[2] if (pv is not None or ov is not None) else 0
    t = torch.empty(B, R, dtype=dtype, device="cuda")
    body, feat = (torch.empty(B, R, dtype=torch.int32, device="cuda") for _ in range(2))
    n = torch.empty(B, R, 2, dtype=dtype, device="cuda") if normal else None
    aw = pack_bits(active.cuda()) if active is not None else None
    rc = lib.lcpb200_raycast(_lib.dtype_code(dtype), B, pos.shape[1], 0 if pv is None else pv.shape[1],
                             0 if ov is None else ov.shape[1], nv, R, max_dist, _lib.ptr(pos), _lib.ptr(rad),
                             _lib.ptr(pv), _lib.ptr(ov), _lib.ptr(o), _lib.ptr(u), _lib.ptr(aw), _lib.ptr(t),
                             _lib.ptr(body), _lib.ptr(feat), _lib.ptr(n), _lib.stream_ptr(torch.device("cuda")))
    assert rc == 0, lib.lcpb200_last_error_string()
    torch.cuda.synchronize()
    return t, body.long(), feat.long(), n


def reference(sc, dtype, max_dist, active=None):
    """ray_ref in fp64 on the scene's values rounded to dtype (on the GPU, in chunks of rays)"""
    dv = lambda k: None if sc[k] is None else sc[k].to(dtype).to("cuda", f64)
    return ray_ref(dv("pos"), dv("rad"), dv("pv"), dv("ov"), dv("o"), dv("u"), max_dist,
                   None if active is None else active.cuda(), chunk=64)


CONFIGS = {                       # nb, npoly, no, V
    "circles": (40, 0, 0, 0),
    "circles_obstacles": (30, 0, 3, 4),
    "mixed_padded": (20, 6, 3, 7),
    "nv256": (8, 9, 2, 256),
}


def check_against_reference(sc, dtype, max_dist, active=None):
    t, body, feat, n = raw(sc, dtype, max_dist, active)
    rt, rb, rf, rn, margin = reference(sc, dtype, max_dist, active)
    if dtype == f64:
        assert bool((margin > 1e-9).all()), float(margin.min())          # seeded scenes: no near tie
        ok = torch.ones_like(margin, dtype=torch.bool)
        # the circle normal (w + t u) / r cancels |w| (up to 100) down to r (1 to 5), and a grazing entry amplifies t's
        # round-off: measured on an H100, at most 3e-11
        tol, tol_n, floor = 1e-12, 1e-10, 1.0
    else:
        # decisions in fp32 arithmetic agree with fp64 ones only away from their thresholds (neighbouring edges of a
        # 256-gon enter at nearly the same t, so those rays are often ambiguous in fp32); coordinates of up to 100 carry
        # 6e-6 of round-off each, so t is compared relative to max(t, 10) and the normal to 1e-3
        # (measured 2.7e-4); ill-conditioned entries (grazing, origin near a surface) that pass the decision filter
        # reach 4.0e-5 in t, hence 1e-4
        ok = margin > 1e-3
        assert float(ok.float().mean()) > 0.5, float(ok.float().mean())
        tol, tol_n, floor = 1e-4, 1e-3, 10.0
    assert torch.equal(body[ok], rb[ok]) and torch.equal(feat[ok], rf[ok])
    scale = rt.abs().clamp_min(floor)
    assert float(((t.double() - rt).abs() / scale)[ok].max()) <= tol
    assert float((n.double() - rn).abs()[ok].max()) <= tol_n
    assert float((rb >= 0).float().mean()) > 0.05                           # the scenes are not empty
    return body


@pytest.mark.parametrize("dtype", [f64, torch.float32])
@pytest.mark.parametrize("B", [1, 300])
@pytest.mark.parametrize("config", list(CONFIGS))
def test_kernel_matches_reference(config, B, dtype):
    nb, np_, no, V = CONFIGS[config]
    R = 600 if B == 1 else 70                                              # 3 CTAs of 256 rays; one of 96 threads
    sc = scene(B, nb, np_, no, V, R, seed=11 + B + 7 * len(config))
    check_against_reference(sc, dtype, 60.0)


@pytest.mark.parametrize("dtype", [f64, torch.float32])
def test_large_world_with_active(dtype):
    """4000 circles (16 tiles), 40 polygons of 256 vertices (10 tiles) and 3 obstacles, random activity"""
    sc = scene(2, 4000, 40, 3, 256, 300, seed=5, L=400.0)
    g = torch.Generator().manual_seed(6)
    active = torch.rand(2, 4043, generator=g) < 0.6
    body = check_against_reference(sc, dtype, 150.0, active)
    hit = body >= 0
    assert bool(active.cuda().gather(1, body.clamp_min(0))[hit].all())     # inactive bodies are never reported


def test_deterministic_and_independent_of_the_split():
    sc = scene(4, 30, 5, 3, 6, 700, seed=21)
    a, b = raw(sc, f64, 60.0), raw(sc, f64, 60.0)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    halves = [raw(dict(sc, o=sc["o"][:, k], u=sc["u"][:, k]), f64, 60.0) for k in (slice(0, 333), slice(333, 700))]
    for x, y0, y1 in zip(a, *halves):
        assert torch.equal(x, torch.cat([y0, y1], 1))
    t, body, feat, _ = raw(sc, f64, 60.0, normal=False)
    assert torch.equal(t, a[0]) and torch.equal(body, a[1]) and torch.equal(feat, a[2])


def test_active_scene_reads_its_standalone_world():
    nb, np_, no = 25, 6, 3
    sc = scene(12, nb, np_, no, 6, 300, seed=31)
    g = torch.Generator().manual_seed(32)
    active = torch.rand(12, nb + np_ + no, generator=g) < 0.5
    t, body, feat, n = raw(sc, f64, 80.0, active)
    for s in range(12):
        idx = active[s].nonzero().squeeze(1)
        ci, pi, oi = idx[idx < nb], idx[(idx >= nb) & (idx < nb + np_)] - nb, idx[idx >= nb + np_] - nb - np_
        sub = dict(pos=sc["pos"][s:s + 1, ci], rad=sc["rad"][s:s + 1, ci],
                   pv=sc["pv"][s:s + 1, pi] if len(pi) else None, ov=sc["ov"][s:s + 1, oi] if len(oi) else None,
                   o=sc["o"][s:s + 1], u=sc["u"][s:s + 1])
        if len(ci) == 0:
            sub["pos"], sub["rad"] = torch.zeros(1, 0, 2, dtype=f64), torch.zeros(1, 0, dtype=f64)
        ts, bs, fs, ns = raw(sub, f64, 80.0)
        mapped = torch.where(bs >= 0, idx.cuda()[bs.clamp_min(0)], -1)
        assert torch.equal(mapped, body[s:s + 1]) and torch.equal(fs, feat[s:s + 1])
        assert float((ts - t[s:s + 1]).abs().max()) <= 1e-14 * 80.0
        assert torch.equal(ns, n[s:s + 1])
    hit = body >= 0
    assert bool(active.cuda().gather(1, body.clamp_min(0))[hit].all())


# ---------------------------------------------------------------------------------------------------- BatchedWorld
def world(sc, **kw):
    from lcp_physics_b200.world import BatchedWorld
    B, nb = sc["pos"].shape[:2]
    return BatchedWorld(sc["pos"], sc["rad"], polygons=sc["pv"], obstacles=sc["ov"], device="cuda",
                        strict_no_penetration=False, contact_capacity=4096, gravity=None, **kw)


def world_scene(seed):
    sc = scene(6, 12, 4, 3, 6, 128, seed=seed)
    return sc


def test_graph_path_equals_kernel_path():
    sc = world_scene(41)
    w = world(sc)
    o, u = sc["o"].cuda(), sc["u"].cuda()
    with torch.no_grad():
        d0, b0, n0 = w.raycast(o, u * 3.0, 60.0)
    og = o.clone().requires_grad_()
    d1, b1, n1 = w.raycast(og, u * 3.0, 60.0)
    assert d1.requires_grad and torch.equal(b0, b1)
    assert float((d1.detach() - d0).abs().max()) <= 1e-14 * 60.0
    assert float((n1.detach() - n0).abs().max()) <= 1e-12                   # circle normals: see above
    assert torch.equal(b0, raw(sc, f64, 60.0)[1])
    # rays shared by the batch ([R, 2]) and a zero direction
    d2, b2, _ = w.raycast(o[0], torch.zeros_like(u[0]), 60.0)
    assert bool((b2 == -1).all()) and bool((d2 == 60.0).all())


def leaves_of(w, sc):
    """the world's state and geometry as leaves, installed in w: origin, direction, p, rad, plocal, ov"""
    o = sc["o"].cuda().clone().requires_grad_()
    d = (1.5 * sc["u"]).cuda().clone().requires_grad_()
    w.p = w.p.detach().clone().requires_grad_()
    w.rad = w.rad.detach().clone().requires_grad_()
    w.plocal = w.plocal.detach().clone().requires_grad_()
    w.ov = w.ov.detach().clone().requires_grad_()
    return [o, d, w.p, w.rad, w.plocal, w.ov]


def test_gradients_against_central_differences():
    # no padding: moving a repeated vertex by h would make a sliver edge of length h, a non-convex polygon
    sc = scene(2, 4, 3, 2, 5, 24, seed=51, L=40.0, pad=False)
    w = world(sc)
    names = ["origin", "direction", "p", "rad", "plocal", "ov"]
    leaves = leaves_of(w, sc)
    attrs = {2: "p", 3: "rad", 4: "plocal", 5: "ov"}

    def readings(vals):
        for k, a in attrs.items():
            setattr(w, a, vals[k])
        return w.raycast(vals[0], vals[1], 60.0)

    d, body, _ = readings(leaves)
    assert int((body >= 0).sum()) >= 15
    with torch.no_grad():
        u = leaves[1] / leaves[1].norm(dim=2, keepdim=True)
        margin = ray_ref(w.p[:, :w.nb, 1:], w.rad, w.polygon_vertices(), w.ov, leaves[0], u, 60.0)[4]
    robust = margin > 1e-4                                                 # rays whose choices a step of h cannot flip
    assert int(robust.sum()) >= 40
    wt = torch.rand(d.shape, generator=torch.Generator().manual_seed(52), dtype=f64).cuda() * robust
    grads = torch.autograd.grad((d * wt).sum(), leaves)
    h = 1e-6
    base = [x.detach() for x in leaves]
    for k, (x, gx) in enumerate(zip(base, grads)):
        flat = x.reshape(-1)
        fd = torch.empty_like(flat)
        with torch.no_grad():
            for i in range(flat.numel()):
                ys = []
                for sgn in (1.0, -1.0):
                    xp = flat.clone()
                    xp[i] += sgn * h
                    vals = list(base)
                    vals[k] = xp.reshape(x.shape)
                    dd, bb, _ = readings(vals)
                    flip = (bb != body) & robust                           # the choices do not move
                    assert not bool(flip.any()), (names[k], i, flip.nonzero().tolist(), margin[flip].tolist(),
                                                  body[flip].tolist(), bb[flip].tolist())
                    ys.append((dd * wt).sum())
                fd[i] = (ys[0] - ys[1]) / (2 * h)
        scale = float(fd.abs().max().clamp_min(1e-3))
        err = float((gx.reshape(-1) - fd).abs().max()) / scale
        assert err < 1e-6, (names[k], err)


def test_jacrev_equals_jacfwd_in_the_state():
    sc = world_scene(61)
    w = world(sc)
    o, u = sc["o"][:, :40].cuda(), sc["u"][:, :40].cuda()
    p0 = w.p.detach().clone()

    def f(p):
        w.p = p
        d, _, n = w.raycast(o, u, 60.0)
        return torch.cat([d, n.reshape(d.shape[0], -1)], 1)

    jr = torch.func.jacrev(f)(p0)
    jf = torch.func.jacfwd(f)(p0)
    assert float(jr.abs().max()) > 0.1
    assert float((jr - jf).abs().max()) <= 1e-10 * float(jr.abs().max())


# ---------------------------------------------------------------------------------------------------- lidar
def bin_world(vel, fric, exact=True, **kw):
    """6 balls per scene sliding on a Rect floor inside a bin of walls, 4 scenes"""
    from lcp_physics_b200.world import BatchedWorld, rect_vertices
    B = vel.shape[0]
    x = torch.tensor([15.0, 30.0, 45.0, 60.0, 75.0, 90.0], dtype=f64)
    pos = torch.stack([x, torch.full_like(x, 65.0)], 1).expand(B, -1, -1) + \
        torch.tensor([[0.0, 0.0]] * 6, dtype=f64)
    obst = torch.stack([rect_vertices([52.5, 75.0], [115.0, 10.0]), rect_vertices([-5.0, 35.0], [10.0, 90.0]),
                        rect_vertices([110.0, 35.0], [10.0, 90.0])])
    return BatchedWorld(pos.contiguous(), torch.full((B, 6), 5.0, dtype=f64), vel=vel, fric_coeff=fric,
                        obstacles=obst, gravity=100.0, dt=1.0 / 60, max_iter=40, exact_adjoint=exact,
                        device="cuda", **kw)


def bin_leaves(B=4):
    g = torch.Generator().manual_seed(71)
    vel = torch.zeros(B, 6, 3, dtype=f64)
    vel[..., 1] = 20.0 * (1 - 2 * (torch.arange(6) % 2)) * (0.5 + torch.rand(B, 6, generator=g, dtype=f64))
    fric = 0.3 + 0.5 * torch.rand(B, 6, generator=g, dtype=f64)
    return vel.cuda(), fric.cuda()


def rollout_lidar(vel, fric, steps=20, exact=True):
    w = bin_world(vel, fric, exact)
    hist = []
    for _ in range(steps):
        w.step()
        hist.append((w.counts.tolist(), w.t.tolist()))
    d, body, _ = w.lidar(2, 32, 80.0, start=0.1)
    return d, body, hist


def test_lidar_rollout_gradients_both_modes():
    """d(weighted lidar readings after 20 steps) / d(initial velocity, friction): reverse mode (exact adjoint) and forward
    mode (forward_ad) against central differences with identical contact and dt-halving history"""
    import torch.autograd.forward_ad as fwAD
    vel0, fric0 = bin_leaves()
    g = torch.Generator().manual_seed(72)
    wt = torch.rand(4, 32, generator=g, dtype=f64).cuda()
    dirs = {"vel": torch.randn(vel0.shape, generator=g, dtype=f64).cuda(),
            "fric": torch.randn(fric0.shape, generator=g, dtype=f64).cuda()}
    dirs["vel"][..., 0] = 0.0
    vel, fric = vel0.clone().requires_grad_(), fric0.clone().requires_grad_()
    d, body, hist = rollout_lidar(vel, fric)
    assert int((body >= 6).sum()) > 10 and int(((body >= 0) & (body < 6)).sum()) > 10   # walls, floor and balls seen
    gv, gf = torch.autograd.grad((d * wt).sum(), [vel, fric])
    rev = {"vel": float((gv * dirs["vel"]).sum()), "fric": float((gf * dirs["fric"]).sum())}
    h = 1e-6
    for name in ("vel", "fric"):
        with torch.no_grad():
            ys = []
            for sgn in (1.0, -1.0):
                args = dict(vel=vel0, fric=fric0)
                args[name] = args[name] + sgn * h * dirs[name]
                dd, bb, hh = rollout_lidar(args["vel"], args["fric"])
                assert hh == hist and torch.equal(bb, body), name
                ys.append(float((dd * wt).sum()))
            fd = (ys[0] - ys[1]) / (2 * h)
            with fwAD.dual_level():
                args = dict(vel=vel0, fric=fric0)
                args[name] = fwAD.make_dual(args[name], dirs[name])
                dd, _, _ = rollout_lidar(args["vel"], args["fric"])
                fwd = float((fwAD.unpack_dual(dd).tangent * wt).sum())
        scale = max(abs(fd), 1e-3)
        assert abs(rev[name] - fd) < 1e-4 * scale, (name, rev[name], fd)
        assert abs(fwd - fd) < 1e-4 * scale, (name, fwd, fd)


def test_lidar_turns_with_its_body():
    sc = world_scene(81)
    w = world(sc)
    n = 48
    for mount in (3, 12):                                                  # a circle and a polygon
        d0, b0, _ = w.lidar(mount, n, 60.0, start=0.2)
        p = w.p.clone()
        p[:, mount, 0] += 2 * math.pi / n
        w.p = p
        d1, b1, _ = w.lidar(mount, n, 60.0, start=0.2)
        assert torch.equal(b1, b0.roll(-1, 1))
        assert float((d1 - d0.roll(-1, 1)).abs().max()) <= 1e-11 * 60.0
        assert not bool((b0 == mount).any())
        assert bool((b0 >= 0).any())


# ---------------------------------------------------------------------------------------------------- the entry point
def test_entry_point_rejects_bad_arguments():
    from lcp_physics_b200 import _lib
    lib = _lib.load()
    z = lambda *s: torch.zeros(*s, dtype=f64, device="cuda")
    pos, rad, pv, o, u = z(2, 3, 2), z(2, 3), z(2, 1, 4, 2), z(2, 5, 2), z(2, 5, 2)
    t, body, feat = z(2, 5), torch.zeros(2, 5, dtype=torch.int32, device="cuda"), torch.zeros(2, 5, dtype=torch.int32,
                                                                                                device="cuda")
    aw = torch.zeros(2, 300, dtype=torch.int32, device="cuda")
    P = _lib.ptr
    good = dict(dtype=1, B=2, nb=3, np=1, no=0, nv=4, R=5, md=10.0, pos=P(pos), rad=P(rad), pv=P(pv), ov=None,
                o=P(o), u=P(u), aw=None, t=P(t), body=P(body), feat=P(feat), n=None)

    def call(**kw):
        a = dict(good, **kw)
        return lib.lcpb200_raycast(a["dtype"], a["B"], a["nb"], a["np"], a["no"], a["nv"], a["R"], a["md"], a["pos"],
                                   a["rad"], a["pv"], a["ov"], a["o"], a["u"], a["aw"], a["t"], a["body"], a["feat"],
                                   a["n"], None)
    assert call() == 0
    torch.cuda.synchronize()
    bad = [dict(B=0), dict(R=0), dict(B=-1), dict(nb=0, np=0), dict(nv=257), dict(nv=2), dict(md=-1.0),
           dict(md=math.inf), dict(md=math.nan), dict(dtype=0, md=1e39), dict(pos=None), dict(rad=None), dict(pv=None),
           dict(no=1), dict(o=None), dict(u=None), dict(t=None), dict(body=None), dict(feat=None),
           dict(nb=8192, aw=P(aw)), dict(B=70000, R=40000), dict(dtype=2)]
    for kw in bad:
        assert call(**kw) != 0, kw
    with pytest.raises(ValueError, match="origin"):
        world(world_scene(91)).raycast(torch.zeros(3, 4, 2), torch.ones(4, 2), 1.0)
    w = world(world_scene(91))
    for args, name in [((torch.zeros(5, 2), torch.ones(4, 2), 1.0), "direction"),
                       ((torch.zeros(5, 3), torch.ones(5, 3), 1.0), "origin"),
                       ((torch.zeros(5, 2, dtype=torch.int64), torch.ones(5, 2), 1.0), "origin"),
                       ((torch.zeros(5, 2), torch.ones(5, 2), -1.0), "max_dist")]:
        with pytest.raises(ValueError, match=name):
            w.raycast(*args)
    for args, name in [((99, 8, 1.0), "body"), ((0, 0, 1.0), "n_rays")]:
        with pytest.raises(ValueError, match=name):
            w.lidar(*args)
