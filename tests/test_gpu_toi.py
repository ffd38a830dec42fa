"""GPU: times of impact between moving, rotating bodies -- lcpb200_time_of_impact, BatchedWorld.time_of_impact /
first_impact, and the continuous-collision step (ccd=True).

* the kernel against the brute-force reference tests/toi_ref.py on seeded scenes (circles; circles and obstacles;
  spinning padded hulls, circles and obstacles; 256-vertex polygons), fp32 and fp64, B in {1, 300}, K across the
  256-query chunk, both modes: choices equal where the reference's margin is wide, tau within tol / |d'| of the
  reference and never after it, normals; every hit is safe (d >= gap at sampled earlier tau) and within tol of gap
  (the tested scenes never reach the iteration cap);
* without rotation and with one body still, first_impact at gap 0 makes sweep's choices;
* the walk: ties across tile boundaries, `active`, shared and per-scene no_contact, determinism and chunking;
* the graph path equals the kernel path, gradients match central differences, jacrev matches jacfwd;
* ccd=True: the thin-wall ball never passes the wall and bounces, a spinning rect does not sweep through a ball, an
  impact-shortened step leaves the pair in find_contacts, a trajectory with nothing closing is bit-for-bit that of
  ccd=False, and linearize() matches central differences;
* the argument checks of the entry point and of both methods.
"""
import math

import pytest
import torch

from tests.toi_ref import poses, toi_ref
from tests.distance_ref import pair_ref

pytestmark = pytest.mark.gpu
f64 = torch.float64

CONFIGS = {"circles": (24, 0, 0, 0), "circles_obstacles": (20, 0, 3, 6), "mixed": (6, 6, 3, 8),
           "nv256": (0, 3, 1, 256)}


def hulls(g, B, n, V, L, sign=1.0, pad=True):
    """n random convex polygons per scene of 3..V vertices (pad=False: V), padded to V by repeating the last vertex;
    sign -1 reverses every other polygon's orientation. Vertex j of a k-gon lies on a circle at angle (j + u / 2) 2 pi / k
    plus a common offset (u uniform in [0, 1)): every turn is at least a quarter of 2 pi / k, so the polygons stay convex
    once rounded to float32 (random angles can fall arbitrarily close together, and the rounded polygon then fails
    BatchedWorld's convexity check)."""
    out = torch.empty(B, n, V, 2, dtype=f64)
    for s in range(B):
        for q in range(n):
            k = int(torch.randint(3, V + 1, (1,), generator=g)) if pad else V
            ang = (torch.arange(k, dtype=f64) + 0.5 * torch.rand(k, generator=g, dtype=f64)) * (2 * math.pi / k)
            ang = ang + 2 * math.pi * float(torch.rand(1, generator=g))
            rr = 3 + 7 * float(torch.rand(1, generator=g))
            v = L * torch.rand(2, generator=g, dtype=f64) + rr * torch.stack([torch.cos(ang), torch.sin(ang)], 1)
            if sign < 0 and q % 2:
                v = v.flip(0)
            out[s, q, :k] = v
            out[s, q, k:] = v[-1]
    return out


def world(B, nb, np_, no, V, seed, L=60.0, dtype=f64, spin=1.0, pad=True, **kw):
    """a seeded world (circles, hulls, obstacles) and a motion [B, nd, 3] of about a quarter of the scene, with up to
    `spin` radians of rotation"""
    from lcp_physics_b200.world import BatchedWorld
    g = torch.Generator().manual_seed(seed)
    pos = L * torch.rand(B, max(nb, 0), 2, generator=g, dtype=f64)
    rad = 1 + 3 * torch.rand(B, nb, generator=g, dtype=f64)
    pv = hulls(g, B, np_, V, L, pad=pad) if np_ else None
    ov = hulls(g, B, no, V, L, sign=-1.0, pad=pad) if no else None
    if nb == 0:
        pos, rad = torch.zeros(B, 0, 2, dtype=f64), torch.zeros(B, 0, dtype=f64)
    w = BatchedWorld(pos.to(dtype), rad.to(dtype), polygons=None if pv is None else pv.to(dtype),
                     obstacles=None if ov is None else ov.to(dtype), device="cuda", strict_no_penetration=False,
                     contact_capacity=256, gravity=None, **kw)
    nd = w.nd
    m = torch.empty(B, nd, 3, dtype=f64)
    m[..., 1:] = (torch.rand(B, nd, 2, generator=g, dtype=f64) - 0.5) * (L / 2)
    m[..., 0] = (torch.rand(B, nd, generator=g, dtype=f64) - 0.5) * 2 * spin
    return w, m.to("cuda", dtype), g


def ref_of(w, motion, queries, gap, first, **kw):
    dv = lambda t: None if t is None else t.detach().double().cpu()
    pv = dv(w.polygon_vertices()) if w.np else None
    pc = dv(w.p[:, w.nb:, 1:]) if w.np else None
    return toi_ref(dv(w.p[:, :w.nb, 1:]), dv(w.rad), pv, pc, dv(w.ov) if w.no else None, dv(motion), queries, gap,
                   first=first, **kw)


def check_against_ref(w, motion, out, queries, gap, first, tol, **kw):
    fr, body, dist, nrm = (t.detach().double().cpu() for t in out[:4])
    r = ref_of(w, motion, queries, gap, first, **kw)
    wide = 0
    for i, q in enumerate(queries):
        s, k = q[0], q[-1]
        if r[4][i] < 1e-3:
            continue
        wide += 1
        assert int(body[s, k]) == r[1][i], (q, float(fr[s, k]), r[0][i])
        if r[1][i] < 0:
            continue
        ulp = 1e-12 if tol < 1e-6 else 1e-5             # round-off of the dtype the kernel ran in (tol: its default)
        slack = 4 * tol / max(r[4][i], 1e-3) + ulp
        assert float(fr[s, k]) <= r[0][i] + ulp and float(fr[s, k]) >= r[0][i] - slack, (q, float(fr[s, k]), r[0][i])
        assert float(dist[s, k]) - gap <= tol * 1.01 + ulp and float(dist[s, k]) - gap >= -ulp
        if float(dist[s, k]) > 1e-3:
            assert float((nrm[s, k] - r[3][i]).abs().max()) < 1e-3 + 1e3 * tol, (q, nrm[s, k], r[3][i])
    return wide


@pytest.mark.parametrize("dtype", [f64, torch.float32])
@pytest.mark.parametrize("config", list(CONFIGS))
@pytest.mark.parametrize("B,K", [(1, 1), (1, 255), (300, 256), (300, 257)])
def test_kernel_matches_reference(config, B, K, dtype):
    nb, np_, no, V = CONFIGS[config]
    w, m, g = world(B, nb, np_, no, V, seed=1000 * list(CONFIGS).index(config) + B + K, dtype=dtype)
    nt = w.nd + w.no
    gap = 0.5
    tol = 1e-9 if dtype == f64 else 1e-4
    pairs = torch.randint(0, nt, (B, K, 2), generator=g)
    pairs[..., 0] = pairs[..., 0] % w.nd                         # a moving first body
    pairs[..., 1] = torch.where(pairs[..., 1] == pairs[..., 0], (pairs[..., 0] + 1) % nt, pairs[..., 1])
    out = w.time_of_impact(pairs, m, gap=gap)
    first = w.first_impact(pairs[..., 0], m, gap=gap)
    for o in (out, first):
        assert o[0].dtype == dtype and tuple(o[0].shape) == (B, K)
        assert bool(((o[0] >= 0) & (o[0] <= 1)).all())
    n = 2 if config == "nv256" else 6
    sample = [(s, k) for s in range(min(B, 3)) for k in range(0, K, max(1, K // 3))][:n]
    wide = check_against_ref(w, m, out, [(s, int(pairs[s, k, 0]), int(pairs[s, k, 1]), k) for s, k in sample], gap,
                             False, tol)
    if config != "nv256":
        wide += check_against_ref(w, m, first, [(s, int(pairs[s, k, 0]), k) for s, k in sample[:3]], gap, True, tol)
    assert wide >= len(sample) // 2
    # pair mode reads the first mode's hit body as its pair: the same tau
    hit = first[1] >= 0
    if bool(hit.any()):
        pc = pairs.cuda()
        again = w.time_of_impact(torch.stack([pc[..., 0], torch.where(hit, first[1], pc[..., 1])], 2), m, gap=gap)
        assert torch.equal(again[0][hit], first[0][hit]) and torch.equal(again[1][hit], first[1][hit])


def test_hits_are_safe_and_reach_the_gap():
    """d(tau') >= gap at sampled tau' in [0, frac] for every hit; d - gap <= tol at the hit (no cap reached)"""
    for config in ("circles_obstacles", "mixed"):
        nb, np_, no, V = CONFIGS[config]
        w, m, _ = world(4, nb, np_, no, V, seed=5)
        nt = w.nd + w.no
        q = torch.arange(w.nd)
        fr, body, dist, _, _, _ = w.first_impact(q, m, gap=0.25)
        hits = (body >= 0).nonzero().tolist()
        assert len(hits) >= 4
        assert float((dist[body >= 0] - 0.25).max()) <= 1e-9
        dv = lambda t: t.detach().cpu()
        pv = dv(w.polygon_vertices()) if w.np else None
        for s, k in hits[:16]:
            for f in torch.linspace(0, 1, 9).tolist():
                t = f * float(fr[s, k])
                c, pvt = poses(dv(w.p[:, :w.nb, 1:]), pv, dv(w.p[:, w.nb:, 1:]) if w.np else None, dv(m), t)
                d, _, _, _ = pair_ref(c[s:s + 1], dv(w.rad)[s:s + 1], None if pvt is None else pvt[s:s + 1],
                                      dv(w.ov)[s:s + 1] if w.no else None, torch.tensor([[[k, int(body[s, k])]]]),
                                      math.inf)
                assert float(d) >= 0.25 - 1e-9, (s, k, t)
        assert nt > 0


def test_first_impact_without_rotation_matches_sweep():
    w, m, g = world(3, 10, 4, 3, 6, seed=9, spin=0.0)
    for k in range(w.nd):
        mk = torch.zeros_like(m)
        mk[:, k] = m[:, k]
        fr, body, _, _, _, _ = w.first_impact([k], mk)
        sf, sb, _, _ = w.sweep([k], m[:, k:k + 1, 1:])
        assert torch.equal(body, sb), k
        assert float((fr - sf).abs().max()) <= 1e-6, k


def test_walk_ties_active_no_contact_determinism_and_chunking():
    from lcp_physics_b200.world import BatchedWorld
    # 300 circles far away, 255 and 256 at (-1, 0) and (1, 0) on both sides of the circle tile edge, the mover 299
    # below them moving up: an exact tie, which goes to the lower index
    nb = 300
    pos = torch.stack([torch.arange(nb, dtype=f64) * 3.0, torch.full((nb,), 1000.0, dtype=f64)], 1)
    pos[255], pos[256], pos[299] = torch.tensor([-1.0, 0.0]), torch.tensor([1.0, 0.0]), torch.tensor([0.0, -30.0])
    pos = pos.unsqueeze(0).repeat(2, 1, 1)
    m = torch.zeros(2, nb, 3, dtype=f64, device="cuda")
    m[:, 299, 2] = 60.0
    mk = lambda **kw: BatchedWorld(pos, torch.ones(2, nb, dtype=f64), device="cuda", gravity=None,
                                   strict_no_penetration=False, contact_capacity=4096, **kw)
    fr, body, *_ = mk().first_impact([299], m)
    assert body[:, 0].tolist() == [255, 255]
    act = torch.ones(2, nb, dtype=torch.bool)
    act[1, 255] = False
    assert mk(active=act).first_impact([299], m)[1][:, 0].tolist() == [255, 256]
    for nc, want in (([(255, 299)], [256, 256]), ([[(255, 299)], [(255, 299), (256, 299)]], [256, -1])):
        assert mk(no_contact=nc).first_impact([299], m)[1][:, 0].tolist() == want, nc
    # determinism and chunking
    sc, mm, _ = world(5, 12, 4, 2, 6, seed=17)
    q = torch.randint(0, sc.nd, (5, 300), generator=torch.Generator().manual_seed(1))
    a = sc.first_impact(q, mm)
    b = sc.first_impact(q, mm)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    for lo, hi in ((0, 1), (0, 37), (100, 300)):
        c = sc.first_impact(q[:, lo:hi], mm)
        assert all(torch.equal(x[:, lo:hi], y) for x, y in zip(a, c))


def leaves_of(w):
    w.p = w.p.detach().clone().requires_grad_()
    w.rad = w.rad.detach().clone().requires_grad_()
    w.plocal = w.plocal.detach().clone().requires_grad_()
    w.ov = w.ov.detach().clone().requires_grad_()
    return [w.p, w.rad, w.plocal, w.ov]


def test_graph_path_equals_kernel_path_and_gradients():
    # unpadded polygons: moving one copy of a repeated vertex would open a new edge, a choice the derivative holds fixed
    w, m, g = world(2, 4, 3, 2, 5, seed=41, L=25.0, spin=1.5, pad=False)
    q = torch.arange(w.nd)
    gap = 0.3
    with torch.no_grad():
        k = w.first_impact(q, m, gap=gap, tol=1e-13)
    mm = m.clone().requires_grad_()
    leaves = leaves_of(w) + [mm]
    gph = w.first_impact(q, mm, gap=gap, tol=1e-13)
    assert gph[0].requires_grad and torch.equal(k[1], gph[1]) and int((k[1] >= 0).sum()) >= 4
    for a, b in zip(k, gph):
        assert float((a - b.detach()).abs().max()) <= 1e-12
    r = ref_of(w, m, [(s, int(i)) for s in range(2) for i in q], gap, True)
    # wide decisions the kernel agrees with, and hits that reached the gap rather than the iteration cap
    robust = torch.tensor([x > 1e-3 for x in r[4]]).reshape(2, -1).cuda() & (k[0] > 0.02)
    robust &= k[1] == torch.tensor(r[1]).reshape(2, -1).cuda()
    robust &= (k[1] < 0) | (k[2] - gap <= 1e-12)

    def readings(vals):
        w.p, w.rad, w.plocal, w.ov = vals[:4]
        fr, body, dist, nrm, pa, pb = w.first_impact(q, vals[4], gap=gap, tol=1e-13)
        return torch.cat([fr.unsqueeze(2), nrm, pa, pb], 2), body
    y, body = readings(leaves)
    wt = torch.rand(y.shape, generator=g, dtype=f64).cuda() * robust.unsqueeze(2)
    assert int(robust.sum()) >= 3
    grads = torch.autograd.grad((y * wt).sum(), leaves)
    h = 1e-6
    base = [x.detach() for x in leaves]
    for i_leaf, (x, gx) in enumerate(zip(base, grads)):
        flat = x.reshape(-1)
        fd = torch.empty_like(flat)
        with torch.no_grad():
            for i in range(flat.numel()):
                ys = []
                for sgn in (1.0, -1.0):
                    xp = flat.clone()
                    xp[i] += sgn * h
                    vals = list(base)
                    vals[i_leaf] = xp.reshape(x.shape)
                    a, bb = readings(vals)
                    assert torch.equal(bb[robust], body[robust])
                    ys.append((a * wt).sum())
                fd[i] = (ys[0] - ys[1]) / (2 * h)
        scale = float(fd.abs().max().clamp_min(1e-3))
        assert float((gx.reshape(-1) - fd).abs().max()) / scale < 1e-5, i_leaf
    # jacrev == jacfwd in the state
    w2, m2, _ = world(3, 6, 4, 2, 6, seed=51, L=40.0)
    p0 = w2.p.detach().clone()

    def f(p):
        w2.p = p
        fr, _, d, n, pa, _ = w2.first_impact(torch.arange(w2.nd), m2, gap=0.2)
        return torch.cat([fr, d, n.reshape(3, -1), pa.reshape(3, -1)], 1)
    jr = torch.func.jacrev(f)(p0)
    jf = torch.func.jacfwd(f)(p0)
    assert float(jr.abs().max()) > 0.1
    assert float((jr - jf).abs().max()) <= 1e-9 * float(jr.abs().max())


# ---------------------------------------------------------------------------------------------------- ccd step
def wall_world(ccd):
    from lcp_physics_b200.world import BatchedWorld, rect_vertices
    wall = rect_vertices([50.0, 50.0], [0.5, 100.0]).unsqueeze(0)            # x in [49.75, 50.25]
    vel = torch.tensor([[[0.0, 900.0, 0.0]]], dtype=f64)                      # 30 per step: more than 2 r + 0.5
    return BatchedWorld(torch.tensor([[[35.0, 50.0]]], dtype=f64), torch.tensor([[5.0]], dtype=f64), vel=vel,
                        obstacles=wall, gravity=None, dt=1.0 / 30, device="cuda", ccd=ccd)


def test_ccd_stops_the_thin_wall_ball_and_it_bounces():
    w = wall_world(True)
    xs = []
    for _ in range(30):
        w.step()
        xs.append(float(w.p[0, 0, 1]))
        assert xs[-1] + 5.0 <= 49.75 + 1e-6, xs
    assert min(float(w.v[0, 1]), xs[-1] - xs[-2]) < 0                         # it bounced back


def test_ccd_spinning_rect_does_not_sweep_through_a_ball():
    from lcp_physics_b200.world import BatchedWorld, rect_vertices
    for ccd in (False, True):
        w = BatchedWorld(torch.tensor([[[0.0, 6.0]]], dtype=f64), torch.tensor([[1.0]], dtype=f64),
                         polygons=rect_vertices([0.0, 0.0], [16.0, 1.0]).unsqueeze(0),
                         poly_vel=torch.tensor([[[60.0, 0.0, 0.0]]], dtype=f64), gravity=None, dt=1.0 / 30,
                         device="cuda", ccd=ccd, strict_no_penetration=False)
        w.step()
        ang = float(w.p[0, 1, 0])
        # the ball's centre relative to the rod's frame: which side of the rod it is on
        side = math.cos(ang) * float(w.p[0, 0, 2]) - math.sin(ang) * float(w.p[0, 0, 1])
        if ccd:
            assert side > 0.5 and ang < 1.5, (ang, side)
        else:
            assert ang == pytest.approx(2.0)                                   # discrete: a full 2 rad, through it


@pytest.mark.parametrize("kind", ["circle-circle", "circle-obstacle", "circle-hull", "hull-hull"])
def test_ccd_impact_leaves_the_pair_in_contact(kind):
    from lcp_physics_b200.world import BatchedWorld, rect_vertices
    box = lambda x, y: rect_vertices([x, y], [2.0, 2.0]).unsqueeze(0)
    kw = dict(gravity=None, dt=0.1, device="cuda", ccd=True, strict_no_penetration=False, eps=0.1)
    if kind == "circle-circle":
        w = BatchedWorld(torch.tensor([[[0.0, 0.0], [10.0, 0.0]]], dtype=f64), torch.ones(1, 2, dtype=f64),
                         vel=torch.tensor([[[0.0, 150.0, 0.0], [0.0, 0.0, 0.0]]], dtype=f64), **kw)
    elif kind == "circle-obstacle":
        w = BatchedWorld(torch.tensor([[[0.0, 0.0]]], dtype=f64), torch.ones(1, 1, dtype=f64),
                         vel=torch.tensor([[[0.0, 150.0, 0.0]]], dtype=f64), obstacles=box(10.0, 0.0), **kw)
    elif kind == "circle-hull":
        w = BatchedWorld(torch.tensor([[[0.0, 0.0]]], dtype=f64), torch.ones(1, 1, dtype=f64),
                         vel=torch.tensor([[[0.0, 150.0, 0.0]]], dtype=f64), polygons=box(10.0, 0.3),
                         poly_vel=torch.tensor([[[0.5, 0.0, 0.0]]], dtype=f64), **kw)
    else:
        w = BatchedWorld(torch.zeros(1, 0, 2, dtype=f64), torch.zeros(1, 0, dtype=f64),
                         polygons=torch.cat([box(0.0, 0.0), box(10.0, 0.3)], 0),
                         poly_vel=torch.tensor([[[0.0, 150.0, 0.0], [0.5, 0.0, 0.0]]], dtype=f64), **kw)
    w.step()
    assert float(w.t[0]) < 0.1                                                # the step ended at the impact
    d = w.distance([[0, 1]], 10.0)[0]
    assert float(d) <= 0.1 and float(d) >= 0.0
    pairs = set(zip(w.c_b1[0, :int(w.counts[0])].tolist(), w.c_b2[0, :int(w.counts[0])].tolist()))
    assert (0, 1) in pairs, (kind, float(d), pairs)


def test_ccd_without_closing_pairs_is_bit_for_bit_the_discrete_step():
    from tests.test_gpu_raycast import bin_leaves, bin_world
    vel, fric = bin_leaves()
    vel = vel * 0.01
    ws = [bin_world(vel, fric, ccd=c) for c in (False, True)]
    for _ in range(10):
        for w in ws:
            w.step()
        assert torch.equal(ws[0].p, ws[1].p) and torch.equal(ws[0].v, ws[1].v) and torch.equal(ws[0].t, ws[1].t)


def test_ccd_linearize_matches_central_differences():
    w = wall_world(True)
    x_next, A, Bu = w.linearize()
    assert float(x_next[0, 1]) < 49.75 - 5.0 + 1e-6
    x0 = torch.cat([w.get_p(), w.v], 1).detach()
    h = 1e-6
    for j in range(A.shape[2]):
        ys = []
        for sgn in (1.0, -1.0):
            w2 = wall_world(True)
            w2.p = (x0[:, :3] + sgn * h * torch.eye(6, dtype=f64, device="cuda")[j, :3]).reshape(1, 1, 3)
            w2.v = x0[:, 3:] + sgn * h * torch.eye(6, dtype=f64, device="cuda")[j, 3:]
            w2.find_contacts()
            w2.step()
            ys.append(torch.cat([w2.get_p(), w2.v], 1))
        fd = (ys[0] - ys[1]) / (2 * h)
        assert float((A[0, :, j] - fd[0]).abs().max()) <= 1e-5 * max(1.0, float(fd.abs().max())), (j, A[0, :, j], fd)


def test_argument_checks():
    from lcp_physics_b200 import _lib
    w, m, _ = world(2, 4, 2, 1, 5, seed=71, L=30.0)
    for kw, msg in [(dict(motion=torch.zeros(2, 3, 3)), "motion"), (dict(gap=-1.0), "gap"),
                    (dict(gap=math.inf), "gap"), (dict(skip=math.nan), "skip"), (dict(tol=-1e-3), "tol"),
                    (dict(motion=torch.full((2, w.nd, 3), math.nan, dtype=f64)), "finite"),
                    (dict(motion=torch.zeros(2, w.nd, 3, dtype=torch.int64)), "floating")]:
        args = dict(motion=m)
        args.update(kw)
        with pytest.raises(ValueError, match=msg):
            w.time_of_impact([[0, 1]], **args)
        with pytest.raises(ValueError, match=msg):
            w.first_impact([0], **args)
    for pairs, msg in [([[0, 0]], "twice"), ([[0, 99]], "range"), (torch.zeros(0, 2, dtype=torch.long), "K >= 1"),
                       ([[0.5, 1.0]], "integer")]:
        with pytest.raises(ValueError, match=msg):
            w.time_of_impact(pairs, m)
    assert w.time_of_impact([[0, 1]], m.reshape(2, -1))[0].shape == (2, 1)
    lib = _lib.load()
    i32 = torch.zeros(2, 1, dtype=torch.int32, device="cuda")
    buf = [torch.zeros(2, 1, 2, dtype=f64, device="cuda") for _ in range(4)]
    args = lambda **o: [o.get("dtype", 1), 2, w.nb, w.np, w.no, w.nv, o.get("K", 1), o.get("gap", 0.0),
                        _lib.ptr(w.p[:, :w.nb, 1:].contiguous()), _lib.ptr(w.rad), _lib.ptr(w.polygon_vertices()),
                        _lib.ptr(w.ov), o.get("pcen", _lib.ptr(w.p[:, w.nb:, 1:].contiguous())),
                        o.get("motion", _lib.ptr(m)), _lib.ptr(i32), _lib.ptr(i32), 0, o.get("skip", 0.0),
                        o.get("tol", 1e-9), None, None, o.get("stride", 0), _lib.ptr(buf[0]), _lib.ptr(i32),
                        _lib.ptr(i32), _lib.ptr(buf[1]), _lib.ptr(buf[2]), _lib.ptr(buf[3]), _lib.stream_ptr(w.device)]
    assert lib.lcpb200_time_of_impact(*args()) == 0
    torch.cuda.synchronize()
    for o in (dict(K=0), dict(gap=-1.0), dict(skip=math.inf), dict(tol=-1.0), dict(motion=None), dict(pcen=None),
              dict(stride=-1), dict(dtype=7)):
        assert lib.lcpb200_time_of_impact(*args(**o)) != 0, o
