"""GPU: distances between BatchedWorld bodies -- lcpb200_body_distance, BatchedWorld.distance and BatchedWorld.nearest.

* the kernel against the brute-force reference tests/distance_ref.py (Minkowski differences and sdf_ref) on seeded
  scenes (circles; circles and obstacles; circles, padded polygons and obstacles; 256-vertex polygons), fp32 and fp64,
  B in {1, 300}, K across the 256-query chunk: dist and normal to 1e-12 (fp64) / 1e-4 (fp32) of max(|d|, 1) outside
  near-ties, and the witnesses: |point_b - point_a| = |d|, and on the two boundaries when separated;
* nearest mode makes the choices of the min over pair mode bit for bit (values to round-off), shared queries equal
  expanded ones, and two calls or another split of the queries are bitwise equal;
* per-scene activity and shared / per-scene no_contact masks;
* the graph path equals the kernel path, gradients match central differences, jacrev matches jacfwd, and a clearance
  loss after a 20-step rollout differentiates in both exact_adjoint settings;
* the argument checks of the entry point and of both methods.
"""
import pytest
import torch

from tests.distance_ref import body_sdf, nearest_ref, pair_ref
from tests.test_gpu_raycast import bin_leaves, bin_world, hulls

pytestmark = pytest.mark.gpu
f64 = torch.float64

# config: (nb, np, no, V); scenes and queries checked against the reference (the Minkowski hulls cost O(V^2) each)
CONFIGS = {"circles": (24, 0, 0, 0), "circles_obstacles": (20, 0, 3, 6), "mixed": (6, 6, 3, 8),
           "nv256": (0, 3, 1, 256)}


def scene(B, nb, np_, no, V, seed, L=60.0):
    g = torch.Generator().manual_seed(seed)
    pos = L * torch.rand(B, nb, 2, generator=g, dtype=f64)
    rad = 1 + 4 * torch.rand(B, nb, generator=g, dtype=f64)
    pv = hulls(g, B, np_, V, L) if np_ else None
    ov = hulls(g, B, no, V, L, sign=-1.0) if no else None
    return dict(pos=pos, rad=rad, pv=pv, ov=ov, nt=nb + np_ + no, g=g)


def raw(sc, dtype, max_dist, ba, bb=None, shared=False, active=None, nc=None, nc_stride=0):
    """lcpb200_body_distance on the scene's tensors (cast to dtype): (dist, body, feat, normal, point_a) on the GPU"""
    from lcp_physics_b200 import _lib
    from lcp_physics_b200.world import pack_bits
    lib = _lib.load()
    dv = lambda k: None if sc[k] is None else sc[k].to("cuda", dtype).contiguous()
    pos, rad, pv, ov = (dv(k) for k in ("pos", "rad", "pv", "ov"))
    B, nb = sc["pos"].shape[:2]
    np_, no = [0 if sc[k] is None else sc[k].shape[1] for k in ("pv", "ov")]
    nv = max([sc[k].shape[2] for k in ("pv", "ov") if sc[k] is not None] + [0])
    K = ba.shape[-1]
    i32 = lambda t: None if t is None else t.to("cuda", torch.int32).contiguous()
    ba, bb = i32(ba), i32(bb)
    aw = pack_bits(active.cuda()) if active is not None else None
    dist = torch.empty(B, K, dtype=dtype, device="cuda")
    body = torch.empty(B, K, dtype=torch.int32, device="cuda")
    feat = torch.empty_like(body)
    normal = torch.empty(B, K, 2, dtype=dtype, device="cuda")
    pa = torch.empty_like(normal)
    _lib.check(lib.lcpb200_body_distance(
        _lib.dtype_code(dtype), B, nb, np_, no, nv, K, max_dist, _lib.ptr(pos), _lib.ptr(rad), _lib.ptr(pv),
        _lib.ptr(ov), _lib.ptr(ba), _lib.ptr(bb), int(shared), _lib.ptr(aw), _lib.ptr(nc), nc_stride,
        _lib.ptr(dist), _lib.ptr(body), _lib.ptr(feat), _lib.ptr(normal), _lib.ptr(pa), None))
    torch.cuda.synchronize()
    return dist, body.long(), feat, normal, pa


def worst(x, mask):
    """the largest entry of x where mask holds, 0 where it holds nowhere"""
    return float(x[mask].max()) if bool(mask.any()) else 0.0


def random_pairs(g, B, K, nt):
    a = torch.randint(0, nt, (B, K), generator=g)
    b = (a + torch.randint(1, nt, (B, K), generator=g)) % nt
    return torch.stack([a, b], 2)


def check_witnesses(sc, rows, pairs, d, n, pa, tol):
    """|pb - pa| = |d| (where the normal is not zero); separated pairs: pa on A's boundary and pb on B's"""
    pb = pa + d.unsqueeze(-1) * n
    nz = n.norm(dim=-1) > 0
    if bool(nz.any()):
        assert float(((pb - pa).norm(dim=-1) - d.abs())[nz].abs().max()) <= tol
    groups = [t for t in (sc["pv"], sc["ov"]) if t is not None]
    polys = torch.cat(groups, 1) if groups else None
    nb = sc["pos"].shape[1]
    sep = d > 0
    for k, x in ((0, pa), (1, pb)):
        s, _, _ = body_sdf(sc["pos"], sc["rad"], polys, nb, rows[sep], pairs[..., k][sep], x[sep])
        if s.numel():
            assert float(s.abs().max()) <= tol, k


@pytest.mark.parametrize("K", [1, 255, 256, 257])
@pytest.mark.parametrize("dtype", [f64, torch.float32])
@pytest.mark.parametrize("B", [1, 300])
@pytest.mark.parametrize("config", list(CONFIGS))
def test_kernel_matches_reference(config, B, dtype, K):
    nb, np_, no, V = CONFIGS[config]
    sc = scene(B, nb, np_, no, V, seed=sum(map(ord, config)) + B + K)
    g, nt = sc["g"], sc["nt"]
    md = 40.0
    tol, robust_at = (1e-12, 1e-9) if dtype == f64 else (1e-4, 1e-3)
    scenes = [0, B - 1] if B > 1 else [0]
    nq = 8 if config == "nv256" else K                       # the Minkowski hulls of 256-gons hold 65536 points
    cut = lambda t: t.cpu()[scenes][:, :nq].double()
    sub = {k: (None if sc[k] is None else sc[k][scenes]) for k in ("pos", "rad", "pv", "ov")}
    pairs = random_pairs(g, B, K, nt)
    for mode in ("pair", "nearest"):
        if mode == "pair":
            d, body, feat, n, pa = raw(sc, dtype, md, pairs[..., 0], pairs[..., 1])
            rd, rhit, rn, rm = pair_ref(sub["pos"], sub["rad"], sub["pv"], sub["ov"], pairs[scenes][:, :nq], md)
            rbody = torch.where(rhit, pairs[scenes][:, :nq, 1], -1)
            qp = pairs[scenes][:, :nq]
        else:
            d, body, feat, n, pa = raw(sc, dtype, md, pairs[..., 0])
            rd, rbody, rn, rm = nearest_ref(sub["pos"], sub["rad"], sub["pv"], sub["ov"], pairs[scenes][:, :nq, 0], md)
            qp = torch.stack([pairs[scenes][:, :nq, 0], body.cpu()[scenes][:, :nq]], 2)
        d, body, n, pa = cut(d), body.cpu()[scenes][:, :nq], cut(n), cut(pa)
        ok = rm > robust_at * rd.abs().clamp_min(1.0)
        if config != "nv256":                     # the faces of a 256-gon sit within round-off of a tie in fp32
            assert float(ok.double().mean()) > 0.8, (mode, float(ok.double().mean()))
        assert torch.equal(body[ok], rbody[ok]), mode
        scale = rd.abs().clamp_min(1.0)
        # the distance is continuous across a near-tie: compared everywhere but at the max_dist boundary
        far = (rd - md).abs() > robust_at * scale
        assert worst((d - rd).abs() / scale, far) <= tol, mode
        assert worst((n - rn).norm(dim=2) / scale, ok) <= tol * 10, mode
        hit = body >= 0
        assert 0 < int(hit.sum()) or K == 1
        assert bool((d[~hit] == md).all()) and bool((n[~hit] == 0).all()) and bool((pa[~hit] == 0).all())
        rows = torch.tensor(scenes).unsqueeze(1).expand_as(body)
        wsub = {k: (None if sc[k] is None else sc[k]) for k in ("pos", "rad", "pv", "ov")}
        check_witnesses(wsub, rows[hit], qp[hit], d[hit], n[hit], pa[hit], tol * 10 * float(scale.max()))


def all_pairs_min(sc, dtype, md, q, **kw):
    """nearest mode restated through pair mode: every (query, j != query) pair, then the first j of the smallest
    distance within max_dist (the rule's tie order)"""
    B, K = q.shape
    nt = sc["nt"]
    cand = torch.arange(nt).expand(B, K, nt)
    qq = q.unsqueeze(2).expand(B, K, nt)
    other = torch.where(cand == qq, (qq + 1) % nt, cand)
    out = raw(sc, dtype, md, qq.reshape(B, -1), other.reshape(B, -1), **kw)
    d, body, feat, n, pa = [t.reshape(B, K, nt, *t.shape[2:]) for t in out]
    allowed = (cand != qq).cuda() & (body >= 0)
    dd = torch.where(allowed, d, torch.inf)
    best = dd.min(2).values
    j = (dd == best.unsqueeze(2)).to(torch.int8).argmax(2)
    hit = torch.isfinite(best)
    take = lambda t: torch.gather(t, 2, j.view(B, K, 1, *([1] * (t.dim() - 3))).expand(B, K, 1, *t.shape[3:])).squeeze(2)
    return (torch.where(hit, take(d), torch.full_like(best, md)), torch.where(hit, take(body), -1),
            torch.where(hit, take(feat), -1), take(n), take(pa))


@pytest.mark.parametrize("dtype", [f64, torch.float32])
def test_nearest_equals_min_over_pairs_and_is_deterministic(dtype):
    sc = scene(5, 8, 5, 3, 7, seed=7, L=40.0)
    sc["pos"][:, 1] = sc["pos"][:, 0]                          # coincident circles: exact ties
    sc["rad"][:, 1] = sc["rad"][:, 0]
    sc["pv"][:, 1] = sc["pv"][:, 0]
    q = torch.arange(sc["nt"]).repeat(3)[:37].expand(5, -1).contiguous()
    ref = all_pairs_min(sc, dtype, 30.0, q)
    out = raw(sc, dtype, 30.0, q)
    # the choices bit for bit; the values to round-off (the compiler contracts the pair arithmetic of the two modes
    # into fused multiply-adds differently, DESIGN.md section 8)
    assert torch.equal(out[1], ref[1]) and torch.equal(out[2], ref[2])
    ulp = 8 * torch.finfo(dtype).eps
    for k in (0, 3, 4):
        a, b = out[k], ref[k]
        assert float(((a - b).abs() / b.abs().clamp_min(1.0)).max()) <= ulp * 40, k
    assert torch.equal(raw(sc, dtype, 30.0, q)[0], out[0])      # two calls
    shared = raw(sc, dtype, 30.0, q[0], shared=True)             # shared queries = expanded ones
    for a, b in zip(out, shared):
        assert torch.equal(a, b)
    split = [raw(sc, dtype, 30.0, q[:, s]) for s in (slice(0, 20), slice(20, None))]
    for k, a in enumerate(out):
        assert torch.equal(a, torch.cat([split[0][k], split[1][k]], 1))
    pairs = random_pairs(sc["g"], 5, 300, sc["nt"])
    p1 = raw(sc, dtype, 30.0, pairs[..., 0], pairs[..., 1])
    p2 = [raw(sc, dtype, 30.0, pairs[:, s, 0], pairs[:, s, 1]) for s in (slice(0, 1), slice(1, None))]
    for k, a in enumerate(p1):
        assert torch.equal(a, torch.cat([p2[0][k], p2[1][k]], 1))


# ---------------------------------------------------------------------------------------------------- BatchedWorld
def world(sc, **kw):
    from lcp_physics_b200.world import BatchedWorld
    return BatchedWorld(sc["pos"], sc["rad"], polygons=sc["pv"], obstacles=sc["ov"], device="cuda",
                        strict_no_penetration=False, contact_capacity=4096, gravity=None, **kw)


def test_active_scene_reads_its_standalone_world():
    from lcp_physics_b200.world import BatchedWorld
    sc = scene(3, 6, 4, 3, 6, seed=11, L=40.0)
    nt = sc["nt"]
    g = torch.Generator().manual_seed(12)
    act = torch.rand(3, nt, generator=g) < 0.7
    act[:, 0] = True
    act[:, 6] = True
    w = world(sc, active=act)
    q = torch.arange(nt)
    d, body, n, pa, pb = w.nearest(q, 50.0)
    dp, bp, _, _, _ = w.distance(torch.stack([q, (q + 1) % nt], 1), 50.0)
    for s in range(3):
        keep = act[s].nonzero().flatten()
        c, pl, ob = keep[keep < 6], keep[(keep >= 6) & (keep < 10)] - 6, keep[keep >= 10] - 10
        ws = BatchedWorld(sc["pos"][s:s + 1, c], sc["rad"][s:s + 1, c], polygons=sc["pv"][s:s + 1, pl],
                          obstacles=sc["ov"][s:s + 1, ob] if len(ob) else None, device="cuda",
                          strict_no_penetration=False, contact_capacity=4096, gravity=None)
        ds, bs, ns, pas, _ = ws.nearest(torch.arange(len(keep)), 50.0)
        mapped = torch.where(bs[0] >= 0, keep.cuda()[bs[0].clamp_min(0)], -1)
        assert torch.equal(body[s, keep], mapped) and torch.equal(d[s, keep], ds[0])
        assert torch.equal(n[s, keep], ns[0]) and torch.equal(pa[s, keep], pas[0])
        off = ~act[s]
        assert bool((body[s][off.cuda()] == -1).all()) and bool((d[s][off.cuda()] == 50.0).all())
        both = (act[s] & act[s][(q + 1) % nt]).cuda()
        assert bool((bp[s][~both] == -1).all())


@pytest.mark.parametrize("per_scene", [False, True])
def test_no_contact_masks_in_nearest_mode(per_scene):
    sc = scene(2, 6, 3, 2, 5, seed=21, L=30.0)
    nt = sc["nt"]
    q = torch.arange(nt)
    w_free = world(sc)
    b0 = w_free.nearest(q, 100.0)[1].cpu()
    # exclude the unmasked nearest body of some queries: the shared list from scene 0, scene 1's own when per scene
    pick = lambda s, qs: sorted({tuple(sorted((i, int(b0[s, i])))) for i in qs})
    pairs = [pick(0, range(4)), pick(1, range(4, 8))] if per_scene else pick(0, range(4))
    w = world(sc, no_contact=pairs)
    d, body, _, _, _ = w.nearest(q, 100.0)
    ex = torch.zeros(2, nt, nt, dtype=torch.bool)
    for s in range(2):
        for i, j in (pairs[s] if per_scene else pairs):
            ex[s, i, j] = ex[s, j, i] = True
    rd, rb, _, rm = nearest_ref(sc["pos"], sc["rad"], w_free.polygon_vertices().cpu(), sc["ov"], q.expand(2, nt),
                                100.0, excluded=ex)
    ok = rm > 1e-9
    assert float(ok.double().mean()) > 0.8
    assert torch.equal(body.cpu()[ok], rb[ok])
    assert float((d.cpu() - rd).abs()[ok].max()) <= 1e-12 * 100
    bc = body.cpu()
    for s in range(2):
        for i in range(nt):
            assert bc[s, i] < 0 or not bool(ex[s, i, bc[s, i]])
    assert int((bc != b0).sum()) >= 3                                # the masks change readings


def leaves_of(w):
    w.p = w.p.detach().clone().requires_grad_()
    w.rad = w.rad.detach().clone().requires_grad_()
    w.plocal = w.plocal.detach().clone().requires_grad_()
    w.ov = w.ov.detach().clone().requires_grad_()
    return [w.p, w.rad, w.plocal, w.ov]


def test_graph_path_equals_kernel_path():
    sc = scene(4, 8, 5, 3, 6, seed=31, L=40.0)
    w = world(sc)
    pairs = random_pairs(sc["g"], 4, 64, sc["nt"])
    q = torch.arange(sc["nt"])
    for call in (lambda: w.distance(pairs, 30.0), lambda: w.nearest(q, 30.0)):
        with torch.no_grad():
            k = call()
        leaves_of(w)
        gph = call()
        assert gph[0].requires_grad and torch.equal(k[1], gph[1])
        for a, b in zip(k, gph):
            assert float((a - b.detach()).abs().max()) <= 1e-12
        w = world(sc)


def test_gradients_against_central_differences():
    # no padding: moving a repeated vertex by h would make a sliver edge of length h
    g = torch.Generator().manual_seed(41)
    sc = scene(2, 4, 3, 2, 5, seed=41, L=25.0)
    sc["pv"] = hulls(g, 2, 3, 5, 25.0, pad=False)
    sc["ov"] = hulls(g, 2, 2, 5, 25.0, sign=-1.0, pad=False)
    w = world(sc)
    nt = sc["nt"]
    pairs = torch.tensor([(i, j) for i in range(nt) for j in range(nt) if i != j])
    names = ["p", "rad", "plocal", "ov"]
    leaves = leaves_of(w)

    def readings(vals):
        for a, v in zip(names, vals):
            setattr(w, a, v)
        d, b, n, pa, pb = w.distance(pairs, 60.0)
        return torch.cat([d.unsqueeze(2), n, pa, pb], 2), b

    y, body = readings(leaves)
    with torch.no_grad():
        _, _, _, rm = pair_ref(w.p[:, :w.nb, 1:].cpu(), w.rad.cpu(), w.polygon_vertices().cpu(), w.ov.cpu(),
                               pairs.expand(2, -1, -1), 60.0)
    robust = (rm > 1e-4).cuda().unsqueeze(2)
    assert float(robust.double().mean()) > 0.8
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
                    yy, bb = readings(vals)
                    assert torch.equal(bb, body)
                    ys.append((yy * wt).sum())
                fd[i] = (ys[0] - ys[1]) / (2 * h)
        scale = float(fd.abs().max().clamp_min(1e-3))
        err = float((gx.reshape(-1) - fd).abs().max()) / scale
        assert err < 1e-6, (names[k], err)


def test_jacrev_equals_jacfwd_in_the_state():
    sc = scene(3, 6, 4, 2, 6, seed=51, L=40.0)
    w = world(sc)
    q = torch.arange(sc["nt"])
    p0 = w.p.detach().clone()

    def f(p):
        w.p = p
        d, _, n, pa, pb = w.nearest(q, 60.0)
        return torch.cat([d.reshape(3, -1), n.reshape(3, -1), pa.reshape(3, -1), pb.reshape(3, -1)], 1)

    jr = torch.func.jacrev(f)(p0)
    jf = torch.func.jacfwd(f)(p0)
    assert float(jr.abs().max()) > 0.1
    assert float((jr - jf).abs().max()) <= 1e-10 * float(jr.abs().max())


def rollout_clearance(vel, fric, exact, steps=20):
    """softplus(2 - distance) of every ball to the floor and to its nearest other body, after 20 steps"""
    w = bin_world(vel, fric, exact)
    hist = []
    for _ in range(steps):
        w.step()
        hist.append((w.counts.tolist(), w.t.tolist()))
    balls = torch.arange(6)
    d, b, _, _, _ = w.distance(torch.stack([balls, torch.full_like(balls, 6)], 1), 200.0)
    dn, bn, _, _, _ = w.nearest(balls, 200.0)
    loss = torch.nn.functional.softplus(2.0 - d) + torch.nn.functional.softplus(2.0 - dn)
    return loss, torch.cat([b, bn], 1), hist


@pytest.mark.parametrize("exact", [True, False])
def test_clearance_rollout_gradients(exact):
    """forward mode against central differences in both settings; reverse mode with the exact adjoint (the reference's
    backward, exact_adjoint=False, drops terms of the step derivative: its gradient is only checked to reach the
    leaves, DESIGN.md section 3.4)"""
    import torch.autograd.forward_ad as fwAD
    vel0, fric0 = bin_leaves()
    g = torch.Generator().manual_seed(61)
    wt = torch.rand(4, 6, generator=g, dtype=f64).cuda()
    dirs = {"vel": torch.randn(vel0.shape, generator=g, dtype=f64).cuda(),
            "fric": torch.randn(fric0.shape, generator=g, dtype=f64).cuda()}
    dirs["vel"][..., 0] = 0.0
    vel, fric = vel0.clone().requires_grad_(), fric0.clone().requires_grad_()
    loss, body, hist = rollout_clearance(vel, fric, exact)
    assert bool((body >= 0).all())
    gv, gf = torch.autograd.grad((loss * wt).sum(), [vel, fric])
    rev = {"vel": float((gv * dirs["vel"]).sum()), "fric": float((gf * dirs["fric"]).sum())}
    h = 1e-6
    for name in ("vel", "fric"):
        with torch.no_grad():
            ys = []
            for sgn in (1.0, -1.0):
                args = dict(vel=vel0, fric=fric0)
                args[name] = args[name] + sgn * h * dirs[name]
                ls, bb, hh = rollout_clearance(args["vel"], args["fric"], exact)
                assert hh == hist and torch.equal(bb, body), name
                ys.append(float((ls * wt).sum()))
            fd = (ys[0] - ys[1]) / (2 * h)
            with fwAD.dual_level():
                args = dict(vel=vel0, fric=fric0)
                args[name] = fwAD.make_dual(args[name], dirs[name])
                ls, _, _ = rollout_clearance(args["vel"], args["fric"], exact)
                fwd = float((fwAD.unpack_dual(ls).tangent * wt).sum())
        scale = max(abs(fd), 1e-3)
        assert abs(fwd - fd) / scale < 1e-4, (name, fwd, fd)
        if exact:
            assert abs(rev[name] - fd) / scale < 1e-4, (name, rev[name], fd)
    assert bool(torch.isfinite(gv).all()) and float(gv.abs().sum()) > 0
    assert bool(torch.isfinite(gf).all()) and float(gf.abs().sum()) > 0


def test_argument_checks():
    from lcp_physics_b200 import _lib
    sc = scene(2, 4, 2, 1, 5, seed=71, L=30.0)
    w = world(sc)
    nt = sc["nt"]
    bad = [([[0, 1.5]], "integer"), (torch.tensor([[0.0, 1.0]]), "integer"), ([[True, False]], "integer"),
           (torch.zeros(0, 2, dtype=torch.int64), "K >= 1"), ([[0, nt]], "out of range"), ([[-1, 0]], "out of range"),
           ([[2, 2]], "twice"), ([0, 1], r"\[K, 2\]"), (torch.zeros(3, 4, 2, dtype=torch.int64), r"\[K, 2\]")]
    for arg, msg in bad:
        with pytest.raises(ValueError, match=msg):
            w.distance(arg, 10.0)
    for arg, msg in [([0.5], "integer"), ([], "K >= 1"), ([nt], "out of range"), ([[0, 1, 2]], r"\[K\]"),
                     (torch.zeros(2, 3, 1, dtype=torch.int64), r"\[K\]")]:
        with pytest.raises(ValueError, match=msg):
            w.nearest(arg, 10.0)
    for md in (-1.0, float("inf"), float("nan")):
        with pytest.raises(ValueError, match="max_dist"):
            w.nearest([0], md)
    assert w.distance([[0, 1]], 100.0)[0].shape == (2, 1)
    assert w.nearest(torch.tensor([[0], [1]], dtype=torch.int32), 100.0)[1].shape == (2, 1)
    # the entry point: rejected without launching
    lib = _lib.load()
    buf = torch.zeros(64, dtype=f64, device="cuda")
    ib = torch.zeros(64, dtype=torch.int32, device="cuda")
    p = _lib.ptr

    def call(**kw):
        a = dict(dtype=_lib.dtype_code(f64), B=1, nb=2, np=0, no=0, nv=0, K=1, md=1.0, pos=p(buf), rad=p(buf),
                 pv=None, ov=None, ba=p(ib), bb=None, shared=0, aw=None, nc=None, st=0, dist=p(buf), body=p(ib),
                 feat=p(ib), normal=p(buf), pa=p(buf))
        a.update(kw)
        return lib.lcpb200_body_distance(*a.values(), None)

    assert call() == 0
    for kw in (dict(B=0), dict(K=0), dict(nb=0), dict(md=-1.0), dict(ba=None), dict(pa=None), dict(normal=None),
               dict(st=-1), dict(dtype=7), dict(np=1, nv=2, pv=p(buf)), dict(B=70000, K=70000)):
        assert call(**kw) != 0, kw
    torch.cuda.synchronize()
