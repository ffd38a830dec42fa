"""GPU: shape casts and sweeps against BatchedWorld scenes -- lcpb200_shapecast, BatchedWorld.shapecast and
BatchedWorld.sweep.

* the kernel against the brute-force reference tests/sweep_ref.py on seeded scenes (circles; circles and obstacles;
  circles, padded polygons and obstacles; 256-vertex polygons), fp32 and fp64, B in {1, 300}, K across the 256-query
  chunk, disk mode with radius 0 and > 0 and body mode: choices equal away from the reference's margins, distances to
  1e-12 (fp64) / 1e-4 (fp32) and normals to 1e-11 / 1e-3 of max(|t|, 1);
* consistency: radius 0 makes raycast's choices; a circle's sweep is the shape cast from its centre with its radius;
  a mover translated by frac d touches the hit body (`distance` of the pair is 0);
* the walk past its tiles: more than 256 circles, polygons over several tiles, exact ties across tile boundaries,
  readings exactly at the limit, `active` at tile edges, shared and per-scene no_contact, determinism and chunking;
* the graph path equals the kernel path, gradients match central differences, jacrev matches jacfwd, a sweep of the
  balls' horizontal velocity after a 20-step rollout differentiates in both exact_adjoint settings, and a ball that
  tunnels through a thin wall in step() is caught by sweep;
* the argument checks of the entry point and of both methods.
"""
import math

import pytest
import torch

from tests.sweep_ref import shapecast_ref, sweep_ref
from tests.test_gpu_raycast import bin_leaves, bin_world, hulls

pytestmark = pytest.mark.gpu
f64 = torch.float64

CONFIGS = {"circles": (24, 0, 0, 0), "circles_obstacles": (20, 0, 3, 6), "mixed": (6, 6, 3, 8),
           "nv256": (0, 3, 1, 256)}


def scene(B, nb, np_, no, V, seed, L=60.0):
    g = torch.Generator().manual_seed(seed)
    pos = L * torch.rand(B, nb, 2, generator=g, dtype=f64)
    rad = 1 + 4 * torch.rand(B, nb, generator=g, dtype=f64)
    pv = hulls(g, B, np_, V, L) if np_ else None
    ov = hulls(g, B, no, V, L, sign=-1.0) if no else None
    return dict(pos=pos, rad=rad, pv=pv, ov=ov, nt=nb + np_ + no, g=g)


def raw(sc, dtype, max_dist, o=None, r=None, bq=None, u=None, lim=None, active=None, nc=None, nc_stride=0):
    """lcpb200_shapecast on the scene's tensors (cast to dtype): (dist, body, feat, normal, point) on the GPU"""
    from lcp_physics_b200 import _lib
    from lcp_physics_b200.world import pack_bits
    lib = _lib.load()
    dv = lambda t: None if t is None else t.to("cuda", dtype).contiguous()
    pos, rad, pv, ov = (dv(sc[k]) for k in ("pos", "rad", "pv", "ov"))
    B, nb = sc["pos"].shape[:2]
    np_, no = [0 if sc[k] is None else sc[k].shape[1] for k in ("pv", "ov")]
    nv = max([sc[k].shape[2] for k in ("pv", "ov") if sc[k] is not None] + [0])
    K = u.shape[1]
    o, r, u, lim = dv(o), dv(r), dv(u), dv(lim)
    bq = None if bq is None else bq.to("cuda", torch.int32).contiguous()
    aw = pack_bits(active.cuda()) if active is not None else None
    dist = torch.empty(B, K, dtype=dtype, device="cuda")
    body = torch.empty(B, K, dtype=torch.int32, device="cuda")
    feat = torch.empty_like(body)
    normal = torch.empty(B, K, 2, dtype=dtype, device="cuda")
    point = torch.empty_like(normal)
    _lib.check(lib.lcpb200_shapecast(
        _lib.dtype_code(dtype), B, nb, np_, no, nv, K, max_dist, _lib.ptr(pos), _lib.ptr(rad), _lib.ptr(pv),
        _lib.ptr(ov), _lib.ptr(o), _lib.ptr(r), _lib.ptr(bq), _lib.ptr(u), _lib.ptr(lim), _lib.ptr(aw), _lib.ptr(nc),
        nc_stride, _lib.ptr(dist), _lib.ptr(body), _lib.ptr(feat), _lib.ptr(normal), _lib.ptr(point), None))
    torch.cuda.synchronize()
    return dist, body.long(), feat, normal, point


def queries(g, B, K, nt, L):
    """disk origins, unit directions and radii, and movers with displacements"""
    o = L * torch.rand(B, K, 2, generator=g, dtype=f64)
    a = 2 * math.pi * torch.rand(B, K, generator=g, dtype=f64)
    u = torch.stack([a.cos(), a.sin()], 2)
    r = 0.5 + 2 * torch.rand(B, K, generator=g, dtype=f64)
    bq = torch.randint(0, nt, (B, K), generator=g)
    disp = u * (L / 2) * torch.rand(B, K, 1, generator=g, dtype=f64)
    return o, u, r, bq, disp


def worst(x, mask):
    return float(x[mask].max()) if bool(mask.any()) else 0.0


@pytest.mark.parametrize("K", [1, 255, 256, 257])
@pytest.mark.parametrize("dtype", [f64, torch.float32])
@pytest.mark.parametrize("B", [1, 300])
@pytest.mark.parametrize("config", list(CONFIGS))
def test_kernel_matches_reference(config, B, dtype, K):
    nb, np_, no, V = CONFIGS[config]
    sc = scene(B, nb, np_, no, V, seed=sum(map(ord, config)) + B + K)
    g, nt = sc["g"], sc["nt"]
    L, md = 60.0, 40.0
    tol, robust_at = (1e-12, 1e-9) if dtype == f64 else (1e-4, 1e-3)
    scenes = [0, B - 1] if B > 1 else [0]
    n = 2 if config == "nv256" else 8                          # queries checked at each end of the list
    cols = sorted(set(list(range(min(n, K))) + list(range(max(K - n, 0), K))))
    sub = {k: (None if sc[k] is None else sc[k][scenes]) for k in ("pos", "rad", "pv", "ov")}
    cut = lambda t: t.cpu()[scenes][:, cols]
    o, u, r, bq, disp = queries(g, B, K, nt, L)
    Ld = disp.norm(dim=2)
    for mode in ("ray", "disk", "body"):
        if mode == "body":
            d, body, _, nrm, _ = raw(sc, dtype, 0.0, bq=bq, u=u, lim=Ld)
            rf, rb, rn, rm = sweep_ref(sub["pos"], sub["rad"], sub["pv"], sub["ov"], cut(bq), cut(disp))
            rd = rf * cut(Ld)
        else:
            rr = r if mode == "disk" else torch.zeros_like(r)
            d, body, _, nrm, _ = raw(sc, dtype, md, o=o, r=rr, u=u)
            rd, rb, rn, rm = shapecast_ref(sub["pos"], sub["rad"], sub["pv"], sub["ov"], cut(o), cut(u), cut(rr), md)
        d, body, nrm = cut(d).double(), cut(body), cut(nrm).double()
        scale = rd.abs().clamp_min(1.0)
        ok = rm > robust_at * scale
        if config != "nv256":
            assert float(ok.double().mean()) > 0.8, (mode, float(ok.double().mean()))
        assert torch.equal(body[ok], rb[ok]), mode
        assert worst((d - rd).abs() / scale, ok) <= tol, mode
        assert worst((nrm - rn).norm(dim=2), ok & (rb >= 0)) <= tol * 10, mode
        miss = body < 0
        assert bool((nrm[miss] == 0).all())


@pytest.mark.parametrize("config", ["circles_obstacles", "mixed"])
def test_radius_zero_makes_raycasts_choices(config):
    from lcp_physics_b200 import _lib
    nb, np_, no, V = CONFIGS[config]
    sc = scene(8, nb, np_, no, V, seed=3)
    o, u, _, _, _ = queries(sc["g"], 8, 300, sc["nt"], 60.0)
    d, body, feat, nrm, _ = raw(sc, f64, 40.0, o=o, r=torch.zeros(8, 300, dtype=f64), u=u)
    lib = _lib.load()
    dv = lambda t: None if t is None else t.to("cuda", f64).contiguous()
    t = torch.empty(8, 300, dtype=f64, device="cuda")
    rb = torch.empty(8, 300, dtype=torch.int32, device="cuda")
    rf = torch.empty_like(rb)
    rn = torch.empty(8, 300, 2, dtype=f64, device="cuda")
    args = [dv(x) for x in (sc["pos"], sc["rad"], sc["pv"], sc["ov"], o, u)]    # alive until the kernel has run
    _lib.check(lib.lcpb200_raycast(_lib.dtype_code(f64), 8, nb, np_, no, V, 300, 40.0, *[_lib.ptr(x) for x in args],
                                   None, _lib.ptr(t), _lib.ptr(rb), _lib.ptr(rf), _lib.ptr(rn), None))
    torch.cuda.synchronize()
    assert torch.equal(body, rb.long())
    poly = body >= nb
    assert torch.equal(feat[poly], rf[poly])
    assert float(((d - t).abs() / t.abs().clamp_min(1.0)).max()) <= 1e-13
    assert float((nrm - rn).abs().max()) <= 1e-12
    assert int((body >= 0).sum()) > 500


# ---------------------------------------------------------------------------------------------------- BatchedWorld
def world(sc, **kw):
    from lcp_physics_b200.world import BatchedWorld
    return BatchedWorld(sc["pos"], sc["rad"], polygons=sc["pv"], obstacles=sc["ov"], device="cuda",
                        strict_no_penetration=False, contact_capacity=4096, gravity=None, **kw)


def test_circle_sweep_is_the_shapecast_from_its_centre():
    sc = scene(3, 8, 4, 3, 6, seed=13, L=40.0)
    nt = sc["nt"]
    pairs = [(0, 1), (2, 9), (3, 13)]
    w = world(sc, no_contact=pairs)
    g = torch.Generator().manual_seed(14)
    ks = torch.arange(8)
    a = 2 * math.pi * torch.rand(3, 8, generator=g, dtype=f64)
    disp = 25.0 * torch.stack([a.cos(), a.sin()], 2).cuda()
    fr, body, nrm, pt = w.sweep(ks, disp)
    assert int((body >= 0).sum()) >= 6
    for k in range(8):
        act = torch.ones(3, nt, dtype=torch.bool)
        act[:, k] = False
        for i, j in pairs:
            if k in (i, j):
                act[:, i + j - k] = False
        wk = world(sc, active=act)
        d, b, n, p = wk.shapecast(w.p[:, k, 1:].unsqueeze(1), disp[:, k:k + 1], w.rad[:, k:k + 1], 25.0)
        assert torch.equal(b[:, 0], body[:, k]), k
        assert float((d[:, 0] / 25.0 - fr[:, k]).abs().max()) <= 1e-12
        hit = b[:, 0] >= 0
        assert worst((n[:, 0] + nrm[:, k]).abs().amax(1), hit) <= 1e-12
        assert worst((p[:, 0] - pt[:, k]).abs().amax(1), hit) <= 1e-12


def test_translated_mover_touches_the_hit_body():
    sc = scene(4, 8, 6, 3, 7, seed=17, L=40.0)
    w = world(sc)
    g = torch.Generator().manual_seed(18)
    nd = w.nd
    a = 2 * math.pi * torch.rand(4, nd, generator=g, dtype=f64)
    disp = 30.0 * torch.stack([a.cos(), a.sin()], 2).cuda()
    ks = torch.arange(nd)
    fr, body, nrm, pt = w.sweep(ks, disp)
    hit = body >= 0
    assert int(hit.sum()) >= 10
    moved = world(sc)
    close, agree = [], []
    for s in range(4):
        for k in range(nd):
            if not bool(hit[s, k]):
                continue
            moved.p = w.p.detach().clone()
            moved.p[s, k, 1:] += fr[s, k] * disp[s, k]
            d, _, n, _, _ = moved.distance(torch.tensor([[k, int(body[s, k])]]), 100.0)
            close.append(abs(float(d[s, 0])))
            agree.append(float((n[s, 0] * nrm[s, k]).sum()))
    assert max(close) <= 1e-9
    assert sum(x > 1 - 1e-6 for x in agree) >= 0.8 * len(agree)  # equal away from vertex-vertex contacts


# ---------------------------------------------------------------------------------------------------- walk limits
def test_walk_limits_ties_limit_and_active():
    """300 circles (two circle tiles) and 40 polygons of 64 vertices (16 per tile): ties across both tile boundaries
    go to the lower index, a reading exactly at the limit is a hit, and an inactive body at a tile edge is skipped"""
    B, nb, np_ = 2, 300, 40
    g = torch.Generator().manual_seed(5)
    pos = torch.stack([torch.arange(nb, dtype=f64) * 10.0, torch.full((nb,), 100.0, dtype=f64)], 1).expand(B, -1, -1)
    pos = pos.clone()
    pos[:, 256] = pos[:, 255]                                  # an exact tie across the circle tile boundary
    rad = torch.ones(B, nb, dtype=f64)
    ang = torch.arange(64, dtype=f64) * 2 * math.pi / 64
    pv = torch.stack([torch.stack([q * 10.0 + 2 * ang.cos(), -100.0 + 2 * ang.sin()], 1) for q in range(np_)])
    pv[16] = pv[15]                                            # ... and across a polygon tile boundary
    pv = pv.expand(B, -1, -1, -1).contiguous()
    sc = dict(pos=pos, rad=rad, pv=pv, ov=None, nt=nb + np_)
    # straight down onto circle 255 / 256 and polygon 15 / 16, radius 0.5; circles 255 and 299 read exactly 8
    o = torch.tensor([[2550.0, 109.5], [150.0, -90.0], [2990.0, 110.0], [2990.0, 110.0]], dtype=f64)
    u = torch.tensor([[0.0, -1.0]] * 4, dtype=f64)
    r = torch.tensor([0.5, 0.5, 1.0, 1.0], dtype=f64)
    for dtype in (f64, torch.float32):
        d, body, _, _, _ = raw(sc, dtype, 8.0, o=o.expand(B, -1, -1), r=r.expand(B, -1), u=u.expand(B, -1, -1))
        assert body[0].tolist() == [255, nb + 15, 299, 299] and d[0, 0] == 8.0 and d[0, 2] == 8.0
        d, body, _, _, _ = raw(sc, dtype, 7.5, o=o.expand(B, -1, -1), r=r.expand(B, -1), u=u.expand(B, -1, -1))
        assert body[0, 2] == -1 and d[0, 2] == 7.5
        act = torch.ones(B, nb + np_, dtype=torch.bool)
        act[1, 255] = False
        act[1, nb + 15] = False
        d, body, _, _, _ = raw(sc, dtype, 8.0, o=o.expand(B, -1, -1), r=r.expand(B, -1), u=u.expand(B, -1, -1),
                               active=act)
        assert body[0].tolist()[:2] == [255, nb + 15] and body[1].tolist()[:2] == [256, nb + 16]
    # the same casts against the reference, over scenes that span the tiles
    o2, u2, r2, _, _ = queries(g, B, 64, nb + np_, 1000.0)
    o2[..., 1] = 200.0 * torch.rand(B, 64, generator=g, dtype=f64) - 100.0
    d, body, _, n, _ = raw(sc, f64, 500.0, o=o2, r=r2, u=u2)
    rd, rb, rn, rm = shapecast_ref(pos, rad, pv, None, o2, u2, r2, 500.0)
    ok = rm > 1e-9 * rd.abs().clamp_min(1.0)
    assert torch.equal(body.cpu()[ok], rb[ok]) and float((d.cpu() - rd).abs()[ok].max()) <= 1e-9
    assert int((rb >= 0).sum()) >= 10


@pytest.mark.parametrize("per_scene", [False, True])
def test_no_contact_masks_and_determinism(per_scene):
    sc = scene(2, 6, 3, 2, 5, seed=21, L=30.0)
    nt = sc["nt"]
    q = torch.arange(nt)
    g = torch.Generator().manual_seed(22)
    a = 2 * math.pi * torch.rand(2, nt, generator=g, dtype=f64)
    disp = (40.0 * torch.stack([a.cos(), a.sin()], 2)).cuda()
    w_free = world(sc)
    b0 = w_free.sweep(q, disp)[1].cpu()
    pick = lambda s, qs: sorted({tuple(sorted((i, int(b0[s, i])))) for i in qs if int(b0[s, i]) >= 0})
    pairs = [pick(0, range(6)), pick(1, range(5, 11))] if per_scene else pick(0, range(6))
    w = world(sc, no_contact=pairs)
    fr, body, _, _ = w.sweep(q, disp)
    ex = torch.zeros(2, nt, nt, dtype=torch.bool)
    for s in range(2):
        for i, j in (pairs[s] if per_scene else pairs):
            ex[s, i, j] = ex[s, j, i] = True
    rf, rb, _, rm = sweep_ref(sc["pos"], sc["rad"], w_free.polygon_vertices().cpu(), sc["ov"], q.expand(2, nt),
                              disp.cpu(), excluded=ex)
    ok = rm > 1e-9
    assert float(ok.double().mean()) > 0.8
    assert torch.equal(body.cpu()[ok], rb[ok])
    assert float((fr.cpu() - rf).abs()[ok].max()) <= 1e-11
    assert int((body.cpu() != b0).sum()) >= 3
    # determinism, and another split of the queries
    again = w.sweep(q, disp)
    parts = [w.sweep(q[s], disp[:, s]) for s in (slice(0, 4), slice(4, None))]
    for k in range(4):
        assert torch.equal(again[k], (fr, body, *again[2:])[k])
        assert torch.equal(again[k], torch.cat([parts[0][k], parts[1][k]], 1))


def test_chunking_is_invisible():
    sc = scene(3, 10, 5, 3, 6, seed=23, L=50.0)
    o, u, r, bq, disp = queries(sc["g"], 3, 600, sc["nt"], 50.0)
    for dtype in (f64, torch.float32):
        kw = dict(o=o, r=r, u=u)
        full = raw(sc, dtype, 40.0, **kw)
        parts = [raw(sc, dtype, 40.0, **{k: v[:, s] for k, v in kw.items()}) for s in (slice(0, 257), slice(257, None))]
        lim = disp.norm(dim=2)
        fb = raw(sc, dtype, 0.0, bq=bq, u=u, lim=lim)
        pb = [raw(sc, dtype, 0.0, bq=bq[:, s], u=u[:, s], lim=lim[:, s]) for s in (slice(0, 33), slice(33, None))]
        for k in range(5):
            assert torch.equal(full[k], torch.cat([parts[0][k], parts[1][k]], 1)), k
            assert torch.equal(fb[k], torch.cat([pb[0][k], pb[1][k]], 1)), k
            assert torch.equal(full[k], raw(sc, dtype, 40.0, **kw)[k]), k


# ---------------------------------------------------------------------------------------------------- derivatives
def leaves_of(w):
    w.p = w.p.detach().clone().requires_grad_()
    w.rad = w.rad.detach().clone().requires_grad_()
    w.plocal = w.plocal.detach().clone().requires_grad_()
    w.ov = w.ov.detach().clone().requires_grad_()
    return [w.p, w.rad, w.plocal, w.ov]


def test_graph_path_equals_kernel_path():
    sc = scene(4, 8, 5, 3, 6, seed=31, L=40.0)
    o, u, r, bq, disp = queries(sc["g"], 4, 64, sc["nt"], 40.0)
    o, u, r, bq, disp = o.cuda(), u.cuda(), r.cuda(), bq.cuda(), disp.cuda()
    w = world(sc)
    for call in (lambda: w.shapecast(o, u, r, 30.0), lambda: w.sweep(bq, disp)):
        with torch.no_grad():
            k = call()
        leaves_of(w)
        gph = call()
        assert gph[0].requires_grad and torch.equal(k[1], gph[1])
        assert int((k[1] >= 0).sum()) > 20
        for a, b in zip(k, gph):
            assert float((a - b.detach()).abs().max()) <= 1e-12
        w = world(sc)


def test_gradients_against_central_differences():
    g = torch.Generator().manual_seed(41)
    sc = scene(2, 4, 3, 2, 5, seed=41, L=25.0)
    sc["pv"] = hulls(g, 2, 3, 5, 25.0, pad=False)
    sc["ov"] = hulls(g, 2, 2, 5, 25.0, sign=-1.0, pad=False)
    w = world(sc)
    nt = sc["nt"]
    o, u, r, _, _ = queries(g, 2, 24, nt, 25.0)
    bq = torch.arange(w.nd).repeat(3)
    a = 2 * math.pi * torch.rand(2, len(bq), generator=g, dtype=f64)
    disp = 20.0 * torch.stack([a.cos(), a.sin()], 2)
    q = [o.cuda(), (u * 1.3).cuda(), r.cuda(), disp.cuda()]
    names = ["p", "rad", "plocal", "ov", "origin", "direction", "radius", "displacement"]
    leaves = leaves_of(w) + [t.clone().requires_grad_() for t in q]

    def readings(vals):
        for nm, v in zip(names[:4], vals[:4]):
            setattr(w, nm, v)
        o_, d_, r_, disp_ = vals[4:]
        t, b1, n1, p1 = w.shapecast(o_, d_, r_, 40.0)
        f, b2, n2, p2 = w.sweep(bq, disp_)
        return torch.cat([t.unsqueeze(2), n1, p1], 2).reshape(-1), torch.cat([f.unsqueeze(2), n2, p2], 2).reshape(-1), \
            torch.cat([b1, b2], 1)

    y1, y2, body = readings(leaves)
    y = torch.cat([y1, y2])
    with torch.no_grad():
        pv = w.polygon_vertices().cpu()
        _, _, _, m1 = shapecast_ref(w.p[:, :w.nb, 1:].cpu(), w.rad.cpu(), pv, w.ov.cpu(), o, u, r, 40.0)
        _, _, _, m2 = sweep_ref(w.p[:, :w.nb, 1:].cpu(), w.rad.cpu(), pv, w.ov.cpu(), bq.expand(2, -1), disp)
    rob = lambda m: (m > 1e-4).unsqueeze(2).expand(-1, -1, 5).reshape(-1)
    robust = torch.cat([rob(m1), rob(m2)]).cuda()
    assert float(robust.double().mean()) > 0.8 and int((body >= 0).sum()) >= 20
    wt = torch.rand(y.shape, generator=g, dtype=f64).cuda() * robust
    grads = torch.autograd.grad((y * wt).sum(), leaves)
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
                    a1, a2, bb = readings(vals)
                    assert torch.equal(bb, body)
                    ys.append((torch.cat([a1, a2]) * wt).sum())
                fd[i] = (ys[0] - ys[1]) / (2 * h)
        scale = float(fd.abs().max().clamp_min(1e-3))
        err = float((gx.reshape(-1) - fd).abs().max()) / scale
        assert err < 1e-5, (names[k], err)                     # central differences of frac = t / |d| at h = 1e-6
        assert float(gx.abs().max()) > 0, names[k]


def test_jacrev_equals_jacfwd_in_the_state():
    sc = scene(3, 6, 4, 2, 6, seed=51, L=40.0)
    w = world(sc)
    o, u, r, _, _ = queries(sc["g"], 3, 16, sc["nt"], 40.0)
    o, u, r = o.cuda(), u.cuda(), r.cuda()
    q = torch.arange(w.nd)
    disp = (20.0 * u[:, :w.nd]).contiguous()
    p0 = w.p.detach().clone()

    def f(p):
        w.p = p
        t, _, n1, p1 = w.shapecast(o, u, r, 60.0)
        fr, _, n2, p2 = w.sweep(q, disp)
        return torch.cat([t, n1.reshape(3, -1), p1.reshape(3, -1), fr, n2.reshape(3, -1), p2.reshape(3, -1)], 1)

    jr = torch.func.jacrev(f)(p0)
    jf = torch.func.jacfwd(f)(p0)
    assert float(jr.abs().max()) > 0.1
    assert float((jr - jf).abs().max()) <= 1e-10 * float(jr.abs().max())


def rollout_sweep(vel, fric, exact, steps=20):
    """frac of each ball's sweep by its horizontal velocity over 60 steps, after 20 steps (the balls roll on the
    floor: their horizontal motion meets the other balls and the walls)"""
    w = bin_world(vel, fric, exact)
    hist = []
    for _ in range(steps):
        w.step()
        hist.append((w.counts.tolist(), w.t.tolist()))
    balls = torch.arange(6)
    vx = w.v.reshape(w.B, w.nd, 3)[:, :, 1]
    fr, body, _, _ = w.sweep(balls, torch.stack([vx, torch.zeros_like(vx)], 2) * (60 * w.dt))
    return fr, body, hist


@pytest.mark.parametrize("exact", [True, False])
def test_sweep_rollout_gradients(exact):
    """forward mode against central differences in both settings; reverse mode with the exact adjoint"""
    import torch.autograd.forward_ad as fwAD
    vel0, fric0 = bin_leaves()
    g = torch.Generator().manual_seed(61)
    wt = torch.rand(4, 6, generator=g, dtype=f64).cuda()
    dirs = {"vel": torch.randn(vel0.shape, generator=g, dtype=f64).cuda(),
            "fric": torch.randn(fric0.shape, generator=g, dtype=f64).cuda()}
    dirs["vel"][..., 0] = 0.0
    vel, fric = vel0.clone().requires_grad_(), fric0.clone().requires_grad_()
    fr, body, hist = rollout_sweep(vel, fric, exact)
    keep = (body >= 0) & (fr > 0.02)                          # hits clear of the start (a fixed choice)
    assert int(keep.sum()) >= 2
    wt = wt * keep
    gv, gf = torch.autograd.grad((fr * wt).sum(), [vel, fric])
    rev = {"vel": float((gv * dirs["vel"]).sum()), "fric": float((gf * dirs["fric"]).sum())}
    h = 1e-6
    for name in ("vel", "fric"):
        with torch.no_grad():
            ys = []
            for sgn in (1.0, -1.0):
                args = dict(vel=vel0, fric=fric0)
                args[name] = args[name] + sgn * h * dirs[name]
                f_, bb, hh = rollout_sweep(args["vel"], args["fric"], exact)
                assert hh == hist and torch.equal(bb[keep], body[keep]), name
                ys.append(float((f_ * wt).sum()))
            fd = (ys[0] - ys[1]) / (2 * h)
            with fwAD.dual_level():
                args = dict(vel=vel0, fric=fric0)
                args[name] = fwAD.make_dual(args[name], dirs[name])
                f_, _, _ = rollout_sweep(args["vel"], args["fric"], exact)
                fwd = float((fwAD.unpack_dual(f_).tangent * wt).sum())
        scale = max(abs(fd), 1e-3)
        assert abs(fwd - fd) / scale < 1e-4, (name, fwd, fd)
        if exact:
            assert abs(rev[name] - fd) / scale < 1e-4, (name, rev[name], fd)
    assert bool(torch.isfinite(gv).all()) and float(gv.abs().sum()) > 0


def test_sweep_catches_a_ball_that_tunnels_through_a_thin_wall():
    from lcp_physics_b200.world import BatchedWorld, rect_vertices
    wall = rect_vertices([50.0, 50.0], [0.5, 100.0]).unsqueeze(0)            # x in [49.75, 50.25]
    vel = torch.tensor([[[0.0, 900.0, 0.0]]], dtype=f64)                      # 30 per step: more than 2 r + 0.5
    w = BatchedWorld(torch.tensor([[[35.0, 50.0]]], dtype=f64), torch.tensor([[5.0]], dtype=f64), vel=vel,
                     obstacles=wall, gravity=None, dt=1.0 / 30, device="cuda")
    fr, body, nrm, pt = w.sweep([0], w.v.reshape(1, 1, 3)[:, :, 1:] * w.dt)
    assert body.tolist() == [[1]]
    assert float(fr[0, 0]) == pytest.approx((49.75 - 5.0 - 35.0) / 30.0, rel=1e-12)
    assert nrm[0, 0].tolist() == pytest.approx([1.0, 0.0]) and pt[0, 0].tolist() == pytest.approx([49.75, 50.0])
    w.step()
    assert float(w.p[0, 0, 1]) > 50.25 + 5.0                                  # discrete detection let it through


def test_argument_checks():
    from lcp_physics_b200 import _lib
    sc = scene(2, 4, 2, 1, 5, seed=71, L=30.0)
    w = world(sc)
    nt = sc["nt"]
    o = torch.zeros(3, 2, dtype=f64)
    u = torch.tensor([[1.0, 0.0]] * 3, dtype=f64)
    for kw, msg in [(dict(origin=torch.zeros(3, 3)), "origin"), (dict(direction=torch.zeros(2, 2)), "as many"),
                    (dict(origin=torch.zeros(3, 2, dtype=torch.int64)), "floating"),
                    (dict(radius=torch.ones(4)), "radius"), (dict(radius=torch.ones(3, 3)), "radius"),
                    (dict(radius=-1.0), "radius"), (dict(radius=float("nan")), "radius"),
                    (dict(max_dist=-1.0), "max_dist"), (dict(max_dist=float("inf")), "max_dist")]:
        a = dict(origin=o, direction=u, radius=1.0, max_dist=10.0)
        a.update(kw)
        with pytest.raises(ValueError, match=msg):
            w.shapecast(**a)
    for b, d, msg in [([0.5], o[:1], "integer"), ([], o[:0], "K >= 1"), ([nt], o[:1], "out of range"),
                      ([[0, 1, 2]], o, r"\[K\]"), ([0, 1], o, "as many"), ([0], torch.zeros(1, 3), "displacement")]:
        with pytest.raises(ValueError, match=msg):
            w.sweep(b, d)
    assert w.shapecast(o, u, torch.ones(2, 3, dtype=f64), 10.0)[0].shape == (2, 3)
    fr, body, nrm, pt = w.sweep([0, 1], torch.zeros(2, 2, dtype=f64))        # no motion: nothing is hit
    assert bool((fr == 1).all()) and bool((body == -1).all()) and bool((nrm == 0).all()) and bool((pt == 0).all())
    # the entry point: rejected without launching; a bad radius in device memory reads a miss
    lib = _lib.load()
    buf = torch.zeros(64, dtype=f64, device="cuda")
    dirb = torch.tensor([1.0, 0.0] * 32, dtype=f64, device="cuda")
    ib = torch.zeros(64, dtype=torch.int32, device="cuda")
    p = _lib.ptr

    def call(**kw):
        a = dict(dtype=_lib.dtype_code(f64), B=1, nb=2, np=0, no=0, nv=0, K=1, md=1.0, pos=p(buf), rad=p(buf),
                 pv=None, ov=None, o=p(buf), r=p(buf), bq=None, u=p(dirb), lim=None, aw=None, nc=None, st=0,
                 dist=p(buf), body=p(ib), feat=p(ib), normal=p(buf), pt=p(buf))
        a.update(kw)
        return lib.lcpb200_shapecast(*a.values(), None)

    assert call() == 0 and call(o=None, r=None, bq=p(ib), lim=p(buf)) == 0
    for kw in (dict(B=0), dict(K=0), dict(nb=0), dict(md=-1.0), dict(md=float("nan")), dict(u=None), dict(o=None),
               dict(r=None), dict(bq=p(ib)), dict(pt=None), dict(normal=None), dict(dist=None), dict(st=-1),
               dict(dtype=7), dict(np=1, nv=2, pv=p(buf)), dict(B=70000, K=70000), dict(nb=9000, aw=p(ib))):
        assert call(**kw) != 0, kw
        msg = lib.lcpb200_last_error_string().decode()
        assert "shapecast" in msg or msg == "bad dtype", (kw, msg)
    torch.cuda.synchronize()
    sc1 = dict(pos=torch.tensor([[[5.0, 0.0]]], dtype=f64), rad=torch.ones(1, 1, dtype=f64), pv=None, ov=None, nt=1)
    for rr in (-0.5, float("nan"), float("inf")):
        d, body, feat, n, pt = raw(sc1, f64, 20.0, o=torch.zeros(1, 1, 2, dtype=f64),
                                   r=torch.tensor([[rr]], dtype=f64), u=torch.tensor([[[1.0, 0.0]]], dtype=f64))
        assert body.tolist() == [[-1]] and feat.tolist() == [[-1]] and d.tolist() == [[20.0]], rr
