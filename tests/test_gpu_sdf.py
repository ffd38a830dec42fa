"""GPU: signed distances and images of BatchedWorld scenes -- lcpb200_signed_distance, BatchedWorld.signed_distance and
BatchedWorld.render.

* the kernel against the brute-force reference tests/sdf_ref.py on seeded scenes (circles only; circles and obstacles;
  circles, padded polygons and obstacles; 256-vertex polygons; a world of thousands of bodies with `active`), fp32 and
  fp64, B in {1, 300}, Q across the 256-point chunk: body and feat equal where the decision margin allows, sdf to
  1e-12 (fp64) / 1e-4 (fp32) of max(|sdf|, 1 / 10), the normal to 1e-10 / 1e-3;
* points shared by the batch equal the same points expanded; determinism and independence of the split;
* the torch mirror (graph path) equals the kernel path, its gradients match central differences (points, state,
  radii, polygon and obstacle vertices, the render window), jacrev matches jacfwd, and a soft-image loss after a
  20-step rollout differentiates in both modes;
* a hard render lights exactly the pixels whose centres lie in the bodies; the entry point and render reject bad
  arguments.
"""
import math

import numpy as np
import pytest
import torch

from tests.sdf_ref import sdf_ref
from tests.test_gpu_raycast import bin_leaves, bin_world, hulls

pytestmark = pytest.mark.gpu
f64 = torch.float64


def scene(B, nb, np_, no, V, Q, seed, L=100.0, pad=True):
    g = torch.Generator().manual_seed(seed)
    pos = L * torch.rand(B, nb, 2, generator=g, dtype=f64)
    rad = 1 + 4 * torch.rand(B, nb, generator=g, dtype=f64)
    pv = hulls(g, B, np_, V, L, pad=pad) if np_ else None
    ov = hulls(g, B, no, V, L, sign=-1.0, pad=pad) if no else None
    x = (L + 20) * torch.rand(B, Q, 2, generator=g, dtype=f64) - 10
    return dict(pos=pos, rad=rad, pv=pv, ov=ov, x=x)


def raw(sc, dtype, max_dist, active=None, normal=True, shared=False):
    """lcpb200_signed_distance on the scene's tensors (cast to dtype): (sdf, body, feat, normal) on the GPU; shared:
    sc["x"] is [Q, 2] and read by every scene"""
    from lcp_physics_b200 import _lib
    from lcp_physics_b200.world import pack_bits
    lib = _lib.load()
    dv = lambda k: None if sc[k] is None else sc[k].to("cuda", dtype).contiguous()
    pos, rad, pv, ov, x = (dv(k) for k in ("pos", "rad", "pv", "ov", "x"))
    B, Q = pos.shape[0], x.shape[-2]
    nv = (pv if pv is not None else ov).shape[2] if (pv is not None or ov is not None) else 0
    sdf = torch.empty(B, Q, dtype=dtype, device="cuda")
    body, feat = (torch.empty(B, Q, dtype=torch.int32, device="cuda") for _ in range(2))
    n = torch.empty(B, Q, 2, dtype=dtype, device="cuda") if normal else None
    aw = pack_bits(active.cuda()) if active is not None else None
    rc = lib.lcpb200_signed_distance(_lib.dtype_code(dtype), B, pos.shape[1], 0 if pv is None else pv.shape[1],
                                     0 if ov is None else ov.shape[1], nv, Q, max_dist, _lib.ptr(pos), _lib.ptr(rad),
                                     _lib.ptr(pv), _lib.ptr(ov), _lib.ptr(x), int(shared), _lib.ptr(aw), _lib.ptr(sdf),
                                     _lib.ptr(body), _lib.ptr(feat), _lib.ptr(n), _lib.stream_ptr(torch.device("cuda")))
    assert rc == 0, lib.lcpb200_last_error_string()
    torch.cuda.synchronize()
    return sdf, body.long(), feat.long(), n


def reference(sc, dtype, max_dist, active=None):
    """sdf_ref in fp64 on the scene's values rounded to dtype (on the GPU, in chunks of points)"""
    dv = lambda k: None if sc[k] is None else sc[k].to(dtype).to("cuda", f64)
    return sdf_ref(dv("pos"), dv("rad"), dv("pv"), dv("ov"), dv("x"), max_dist,
                   None if active is None else active.cuda(), chunk=64)


CONFIGS = {                       # nb, npoly, no, V
    "circles": (40, 0, 0, 0),
    "circles_obstacles": (30, 0, 3, 4),
    "mixed_padded": (20, 6, 3, 7),
    "nv256": (8, 9, 2, 256),
}


def check_against_reference(sc, dtype, max_dist, active=None):
    s, body, feat, n = raw(sc, dtype, max_dist, active)
    rs, rb, rf, rn, margin = reference(sc, dtype, max_dist, active)
    if dtype == f64:
        ok = margin > 1e-9
        assert float(ok.float().mean()) > 0.99, float(ok.float().mean())
        tol, tol_n, floor = 1e-12, 1e-10, 1.0
    else:
        # decisions in fp32 arithmetic agree with fp64 ones only away from their thresholds; coordinates of up to 110
        # carry 7e-6 of round-off each, so sdf is compared relative to max(|sdf|, 10)
        ok = margin > 1e-3
        assert float(ok.float().mean()) > 0.5, float(ok.float().mean())
        tol, tol_n, floor = 1e-4, 1e-3, 10.0
    assert torch.equal(body[ok], rb[ok]) and torch.equal(feat[ok], rf[ok])
    err = float(((s.double() - rs).abs() / rs.abs().clamp_min(floor))[ok].max())
    # (x - q) / |x - q| outside a polygon loses |x| eps / |x - q| to cancellation next to its surface: the normal is
    # compared where |sdf| > 1e-3
    err_n = float((n.double() - rn).abs()[ok & (rs.abs() > 1e-3)].max())
    print("sdf accuracy %s: sdf %.3g, normal %.3g, decided %.4f" % (dtype, err, err_n, float(ok.float().mean())))
    assert err <= tol and err_n <= tol_n, (err, err_n)
    assert float((rb >= 0).float().mean()) > 0.05                           # the scenes are not empty
    assert bool((rs < 0).any())                                             # some points lie inside a body
    return body


@pytest.mark.parametrize("dtype", [f64, torch.float32])
@pytest.mark.parametrize("B", [1, 300])
@pytest.mark.parametrize("config", list(CONFIGS))
def test_kernel_matches_reference(config, B, dtype):
    nb, np_, no, V = CONFIGS[config]
    Q = 1000 if B == 1 else 70                                             # 4 CTAs of 256 points; one of 96 threads
    sc = scene(B, nb, np_, no, V, Q, seed=13 + B + 7 * len(config))
    check_against_reference(sc, dtype, 60.0)


@pytest.mark.parametrize("Q", [1, 255, 256, 257, 1000])
def test_point_counts_across_the_chunk(Q):
    sc = scene(3, 20, 6, 3, 7, Q, seed=100 + Q)
    for dtype in (f64, torch.float32):
        s, body, feat, n = raw(sc, dtype, 60.0)
        rs, rb, rf, _, margin = reference(sc, dtype, 60.0)
        ok = margin > (1e-9 if dtype == f64 else 1e-3)
        assert torch.equal(body[ok], rb[ok]) and torch.equal(feat[ok], rf[ok])
        e = ((s.double() - rs).abs() / rs.abs().clamp_min(10.0))[ok]
        assert e.numel() == 0 or float(e.max()) <= 1e-4


@pytest.mark.parametrize("dtype", [f64, torch.float32])
def test_large_world_with_active(dtype):
    """4000 circles (16 tiles), 40 polygons of 256 vertices (10 tiles) and 3 obstacles, random activity"""
    sc = scene(2, 4000, 40, 3, 256, 300, seed=5, L=400.0)
    g = torch.Generator().manual_seed(6)
    active = torch.rand(2, 4043, generator=g) < 0.6
    body = check_against_reference(sc, dtype, 150.0, active)
    hit = body >= 0
    assert bool(active.cuda().gather(1, body.clamp_min(0))[hit].all())     # inactive bodies are never reported


def test_shared_points_equal_expanded_points():
    sc = scene(5, 20, 6, 3, 7, 600, seed=17)
    xs = sc["x"][0]
    a = raw(dict(sc, x=xs), f64, 60.0, shared=True)
    b = raw(dict(sc, x=xs.expand(5, -1, -1)), f64, 60.0)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_deterministic_and_independent_of_the_split():
    sc = scene(4, 30, 5, 3, 6, 700, seed=21)
    a, b = raw(sc, f64, 60.0), raw(sc, f64, 60.0)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    halves = [raw(dict(sc, x=sc["x"][:, k]), f64, 60.0) for k in (slice(0, 350), slice(350, 700))]
    for x, y0, y1 in zip(a, *halves):
        assert torch.equal(x, torch.cat([y0, y1], 1))
    s, body, feat, _ = raw(sc, f64, 60.0, normal=False)
    assert torch.equal(s, a[0]) and torch.equal(body, a[1]) and torch.equal(feat, a[2])


# ---------------------------------------------------------------------------------------------------- BatchedWorld
def world(sc, **kw):
    from lcp_physics_b200.world import BatchedWorld
    return BatchedWorld(sc["pos"], sc["rad"], polygons=sc["pv"], obstacles=sc["ov"], device="cuda",
                        strict_no_penetration=False, contact_capacity=4096, gravity=None, **kw)


def test_graph_path_equals_kernel_path():
    sc = scene(6, 12, 4, 3, 6, 300, seed=41)
    w = world(sc)
    x = sc["x"].cuda()
    with torch.no_grad():
        s0, b0, n0 = w.signed_distance(x, 60.0)
    xg = x.clone().requires_grad_()
    s1, b1, n1 = w.signed_distance(xg, 60.0)
    assert s1.requires_grad and torch.equal(b0, b1)
    assert float((s1.detach() - s0).abs().max()) <= 1e-12 * 60.0
    assert float((n1.detach() - n0).abs()[s0.abs() > 1e-3].max()) <= 1e-12
    assert torch.equal(b0, raw(dict(sc, pv=w.polygon_vertices().cpu()), f64, 60.0)[1])
    assert bool((b0 >= w.nb).any()) and bool((s0 < 0).any())
    # points shared by the batch ([Q, 2])
    s2, b2, _ = w.signed_distance(x[0], 60.0)
    s3, b3, _ = w.signed_distance(x[0].expand(6, -1, -1), 60.0)
    assert torch.equal(s2, s3) and torch.equal(b2, b3)


def leaves_of(w, sc):
    """the world's state and geometry as leaves, installed in w: points, p, rad, plocal, ov"""
    x = sc["x"].cuda().clone().requires_grad_()
    w.p = w.p.detach().clone().requires_grad_()
    w.rad = w.rad.detach().clone().requires_grad_()
    w.plocal = w.plocal.detach().clone().requires_grad_()
    w.ov = w.ov.detach().clone().requires_grad_()
    return [x, w.p, w.rad, w.plocal, w.ov]


def central_differences(f, leaves, h=1e-6):
    base = [x.detach() for x in leaves]
    out = []
    for k, x in enumerate(base):
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
                    ys.append(f(vals))
                fd[i] = (ys[0] - ys[1]) / (2 * h)
        out.append(fd)
    return out


def test_gradients_against_central_differences():
    # no padding: moving a repeated vertex by h would make a sliver edge of length h, a non-convex polygon
    sc = scene(2, 4, 3, 2, 5, 40, seed=51, L=40.0, pad=False)
    w = world(sc)
    names = ["points", "p", "rad", "plocal", "ov"]
    leaves = leaves_of(w, sc)
    attrs = {1: "p", 2: "rad", 3: "plocal", 4: "ov"}

    def readings(vals):
        for k, a in attrs.items():
            setattr(w, a, vals[k])
        return w.signed_distance(vals[0], 30.0)

    s, body, n = readings(leaves)
    with torch.no_grad():
        margin = sdf_ref(w.p[:, :w.nb, 1:], w.rad, w.polygon_vertices(), w.ov, leaves[0], 30.0)[4]
    robust = margin > 1e-4                                                 # points whose choices a step of h cannot flip
    assert int(robust.sum()) >= 60 and bool((body >= w.nb).any()) and bool((s < 0).any())
    g = torch.Generator().manual_seed(52)
    wt = torch.rand(2, 40, 3, generator=g, dtype=f64).cuda() * robust.unsqueeze(2)
    loss = lambda s, n: (torch.cat([s.unsqueeze(2), n], 2) * wt).sum()
    grads = torch.autograd.grad(loss(s, n), leaves)

    def f(vals):
        ss, bb, nn = readings(vals)
        assert not bool(((bb != body) & robust).any())                     # the choices do not move
        return loss(ss, nn)
    for name, gx, fd in zip(names, grads, central_differences(f, leaves)):
        scale = float(fd.abs().max().clamp_min(1e-3))
        err = float((gx.reshape(-1) - fd).abs().max()) / scale
        assert err < 1e-6, (name, err)


def test_render_window_gradients():
    """d(soft image) / d(lo, hi) of a per-scene window, against central differences"""
    sc = scene(2, 6, 2, 2, 5, 1, seed=53, L=40.0, pad=False)
    w = world(sc)
    lo = torch.tensor([[2.0, 3.0], [5.0, 1.0]], dtype=f64, device="cuda", requires_grad=True)
    hi = torch.tensor([[38.0, 35.0], [36.0, 39.0]], dtype=f64, device="cuda", requires_grad=True)
    wt = torch.rand(2, 12, 16, generator=torch.Generator().manual_seed(54), dtype=f64).cuda()
    img, body, _ = w.render(12, 16, lo, hi, sigma=1.5, max_dist=80.0)
    assert bool((body >= 0).all())
    grads = torch.autograd.grad((img * wt).sum(), [lo, hi])

    def f(vals):
        im, bb, _ = w.render(12, 16, vals[0], vals[1], sigma=1.5, max_dist=80.0)
        return (im * wt).sum()
    for name, gx, fd in zip(["lo", "hi"], grads, central_differences(f, [lo, hi])):
        err = float((gx.reshape(-1) - fd).abs().max()) / float(fd.abs().max().clamp_min(1e-3))
        assert err < 1e-6, (name, err)


def test_jacrev_equals_jacfwd_in_the_state():
    sc = scene(6, 12, 4, 3, 6, 40, seed=61)
    w = world(sc)
    x = sc["x"].cuda()
    p0 = w.p.detach().clone()

    def f(p):
        w.p = p
        s, _, n = w.signed_distance(x, 60.0)
        return torch.cat([s, n.reshape(s.shape[0], -1)], 1)

    jr = torch.func.jacrev(f)(p0)
    jf = torch.func.jacfwd(f)(p0)
    assert float(jr.abs().max()) > 0.1
    assert float((jr - jf).abs().max()) <= 1e-10 * float(jr.abs().max())


def test_hard_render_of_a_circle_and_a_box():
    from lcp_physics_b200.world import BatchedWorld, rect_vertices
    cx, cy, r = 10.3, 12.7, 5.1
    x0, x1, y0, y1 = 20.25, 30.75, 4.25, 9.75
    box = rect_vertices([(x0 + x1) / 2, (y0 + y1) / 2], [x1 - x0, y1 - y0]).unsqueeze(0)
    w = BatchedWorld(torch.tensor([[[cx, cy]]], dtype=f64), torch.tensor([[r]], dtype=f64), obstacles=box,
                     device="cuda", gravity=None)
    H, W = 24, 40
    img, body, sdf = w.render(H, W, (0.0, 0.0), (float(W), float(H)))       # the reference's screen pixels
    X, Y = np.meshgrid(np.arange(W) + 0.5, np.arange(H) + 0.5)               # row i is y = i + 1/2
    in_c = (X - cx) ** 2 + (Y - cy) ** 2 <= r * r
    in_b = (X >= x0) & (X <= x1) & (Y >= y0) & (Y <= y1)
    assert img.shape == (1, H, W) and img.dtype == f64 and not img.requires_grad
    assert np.array_equal(img[0].cpu().numpy() == 1.0, in_c | in_b)
    assert bool((img[0] == 0).cpu().numpy()[~(in_c | in_b)].all())
    b = body[0].cpu().numpy()
    assert (b[in_c] == 0).all() and (b[in_b] == 1).all()
    assert int(in_c.sum()) > 50 and int(in_b.sum()) > 30
    assert float(sdf.max()) <= math.hypot(W, H)


def rollout_image(vel, fric, exact, steps=20):
    w = bin_world(vel, fric, exact)
    hist = []
    for _ in range(steps):
        w.step()
        hist.append((w.counts.tolist(), w.t.tolist()))
    img, body, _ = w.render(24, 32, (-10.0, -5.0), (120.0, 85.0), sigma=2.0, max_dist=200.0)
    return img, body, hist


@pytest.mark.parametrize("exact", [True, False])
def test_soft_image_rollout_gradients(exact):
    """d(weighted soft image after 20 steps) / d(initial velocity, friction): forward mode (forward_ad) against central
    differences with identical contact and dt-halving history in both settings, and reverse mode with the exact
    adjoint. exact_adjoint=False is the reference's backward, which drops terms of the step's derivative (measured 0.66
    and 3.4 relative off the velocity and friction derivatives here): its reverse gradient is only checked to reach the leaves."""
    import torch.autograd.forward_ad as fwAD
    vel0, fric0 = bin_leaves()
    g = torch.Generator().manual_seed(73)
    wt = torch.rand(4, 24, 32, generator=g, dtype=f64).cuda()
    dirs = {"vel": torch.randn(vel0.shape, generator=g, dtype=f64).cuda(),
            "fric": torch.randn(fric0.shape, generator=g, dtype=f64).cuda()}
    dirs["vel"][..., 0] = 0.0
    vel, fric = vel0.clone().requires_grad_(), fric0.clone().requires_grad_()
    img, body, hist = rollout_image(vel, fric, exact)
    assert int((body >= 6).sum()) > 100 and int(((body >= 0) & (body < 6)).sum()) > 50    # walls, floor and balls
    gv, gf = torch.autograd.grad((img * wt).sum(), [vel, fric])
    rev = {"vel": float((gv * dirs["vel"]).sum()), "fric": float((gf * dirs["fric"]).sum())}
    h = 1e-6
    for name in ("vel", "fric"):
        with torch.no_grad():
            ys = []
            for sgn in (1.0, -1.0):
                args = dict(vel=vel0, fric=fric0)
                args[name] = args[name] + sgn * h * dirs[name]
                im, bb, hh = rollout_image(args["vel"], args["fric"], exact)
                assert hh == hist and torch.equal(bb, body), name
                ys.append(float((im * wt).sum()))
            fd = (ys[0] - ys[1]) / (2 * h)
            with fwAD.dual_level():
                args = dict(vel=vel0, fric=fric0)
                args[name] = fwAD.make_dual(args[name], dirs[name])
                im, _, _ = rollout_image(args["vel"], args["fric"], exact)
                fwd = float((fwAD.unpack_dual(im).tangent * wt).sum())
        scale = max(abs(fd), 1e-3)
        print("soft image rollout exact=%s %s: reverse %.3g, forward %.3g (relative to fd)"
              % (exact, name, abs(rev[name] - fd) / scale, abs(fwd - fd) / scale))
        assert abs(fwd - fd) < 1e-4 * scale, (name, fwd, fd)
        if exact:
            assert abs(rev[name] - fd) < 1e-4 * scale, (name, rev[name], fd)
        else:
            assert math.isfinite(rev[name]) and rev[name] != 0.0, (name, rev[name])


# ---------------------------------------------------------------------------------------------------- the entry point
def test_entry_point_rejects_bad_arguments():
    from lcp_physics_b200 import _lib
    lib = _lib.load()
    z = lambda *s: torch.zeros(*s, dtype=f64, device="cuda")
    pos, rad, pv, x = z(2, 3, 2), z(2, 3), z(2, 1, 4, 2), z(2, 5, 2)
    s, body, feat = z(2, 5), torch.zeros(2, 5, dtype=torch.int32, device="cuda"), torch.zeros(2, 5, dtype=torch.int32,
                                                                                                device="cuda")
    aw = torch.zeros(2, 300, dtype=torch.int32, device="cuda")
    P = _lib.ptr
    good = dict(dtype=1, B=2, nb=3, np=1, no=0, nv=4, Q=5, md=10.0, pos=P(pos), rad=P(rad), pv=P(pv), ov=None,
                x=P(x), shared=0, aw=None, s=P(s), body=P(body), feat=P(feat), n=None)

    def call(**kw):
        a = dict(good, **kw)
        return lib.lcpb200_signed_distance(a["dtype"], a["B"], a["nb"], a["np"], a["no"], a["nv"], a["Q"], a["md"],
                                           a["pos"], a["rad"], a["pv"], a["ov"], a["x"], a["shared"], a["aw"], a["s"],
                                           a["body"], a["feat"], a["n"], None)
    assert call() == 0 and call(shared=1) == 0
    torch.cuda.synchronize()
    bad = [dict(B=0), dict(Q=0), dict(B=-1), dict(nb=0, np=0), dict(nv=257), dict(nv=2), dict(md=-1.0),
           dict(md=math.inf), dict(md=math.nan), dict(dtype=0, md=1e39), dict(pos=None), dict(rad=None), dict(pv=None),
           dict(no=1), dict(x=None), dict(s=None), dict(body=None), dict(feat=None), dict(nb=8192, aw=P(aw)),
           dict(B=70000, Q=40000), dict(dtype=2)]
    for kw in bad:
        assert call(**kw) != 0, kw
    w = world(scene(3, 4, 2, 1, 5, 1, seed=91))
    for args, name in [((torch.zeros(4, 5, 2), 1.0), "points"), ((torch.zeros(5, 3), 1.0), "points"),
                       ((torch.zeros(5, 2, dtype=torch.int64), 1.0), "points"), ((torch.zeros(0, 2), 1.0), "points"),
                       ((torch.zeros(5, 2), -1.0), "max_dist"), ((torch.zeros(5, 2), math.nan), "max_dist")]:
        with pytest.raises(ValueError, match=name):
            w.signed_distance(*args)
    lo, hi = (0.0, 0.0), (10.0, 10.0)
    for args, kw, name in [((0, 4, lo, hi), {}, "height"), ((4, 2.5, lo, hi), {}, "width"),
                           ((4, True, lo, hi), {}, "width"), ((4, 4, (0.0, 0.0, 0.0), hi), {}, "lo"),
                           ((4, 4, lo, torch.zeros(5, 2)), {}, "hi"), ((4, 4, lo, (10.0, 0.0)), {}, "lo < hi"),
                           ((4, 4, lo, hi), dict(sigma=-1.0), "sigma"), ((4, 4, lo, hi), dict(sigma=math.inf), "sigma"),
                           ((30000, 30000, lo, hi), {}, "int32")]:
        with pytest.raises(ValueError, match=name):
            w.render(*args, **kw)
