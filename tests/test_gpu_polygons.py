"""GPU: dynamic convex polygons in BatchedWorld (`polygons=`): the hull-hull and circle-polygon contact walk
(lcpb200_contacts with feat) against the CPU oracle (oracle/polygon_oracle.py) on seeded random scenes, the torch
geometry rebuilt from the kernel's features against the kernel's, trajectories recorded from the unmodified reference
(tests/golden/bworld_polygons.npz), a mixed scene on the banded kernel, rollout gradients and fp32."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from oracle.polygon_oracle import OracleHullWorld

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bworld_polygons.npz")
f64 = torch.float64


def _rect(cx, cy, w, h, a):
    c, s = math.cos(a), math.sin(a)
    loc = [(w / 2, h / 2), (-w / 2, h / 2), (-w / 2, -h / 2), (w / 2, -h / 2)]
    return [[cx + c * x - s * y, cy + s * x + c * y] for x, y in loc]


def _hull(cx, cy, r, n, a, g):
    """a convex n-gon of positive area (random radii / angles), padded by repeating its last vertex to 6"""
    ang = sorted(float(t) for t in torch.rand(n, generator=g) * 2 * math.pi)
    pts = [[cx + r * (0.7 + 0.3 * float(torch.rand(1, generator=g))) * math.cos(t + a),
            cy + r * (0.7 + 0.3 * float(torch.rand(1, generator=g))) * math.sin(t + a)] for t in ang]
    v = torch.tensor(pts, dtype=f64)
    from scipy.spatial import ConvexHull
    hv = v[torch.as_tensor(ConvexHull(v.numpy()).vertices)]                          # counter-clockwise: area > 0
    return hv.tolist() + [hv[-1].tolist()] * (6 - hv.shape[0])


def random_scene(seed, nc, npoly, no, spread):
    """circles, rotated boxes and hulls (V = 6), obstacles: overlapping deep and shallow, edge-on (faces nearly
    parallel, 1e-3 apart in angle) and corner-on poses"""
    g = torch.Generator().manual_seed(seed)
    r = lambda: float(torch.rand(1, generator=g))
    pad6 = lambda v: v + [v[-1]] * 2
    circles = [[spread * r(), spread * r()] for _ in range(nc)]
    polys = []
    for k in range(npoly):
        x, y = spread * r(), spread * r()
        kind = k % 4
        if kind == 0:
            polys.append(pad6(_rect(x, y, 10 + 20 * r(), 6 + 14 * r(), 2 * math.pi * r())))
        elif kind == 1:                                                            # edge-on: nearly axis-aligned
            polys.append(pad6(_rect(x, y, 12 + 10 * r(), 8 + 6 * r(), 1e-3 * (1 + r()) * (1 if r() > 0.5 else -1))))
        elif kind == 2:                                                            # corner-on
            polys.append(pad6(_rect(x, y, 14, 14, math.pi / 4 + 0.01 * (r() - 0.5))))
        else:
            polys.append(_hull(x, y, 8 + 8 * r(), 3 + int(4 * r()), 2 * math.pi * r(), g))
    obst = []
    for k in range(no):
        o = _rect(spread * r(), spread * r(), 30 + 40 * r(), 8 + 8 * r(), 0.5 * (r() - 0.5))
        obst.append(pad6(o[::-1] if k % 2 else o))                                    # either orientation
    return dict(pos=torch.tensor(circles, dtype=f64).reshape(nc, 2), rad=torch.tensor([4 + 6 * r() for _ in range(nc)],
                dtype=f64), polys=torch.tensor(polys, dtype=f64).reshape(npoly, 6, 2),
                obst=torch.tensor(obst, dtype=f64).reshape(no, 6, 2),
                pfric=torch.tensor([0.2 + 0.6 * r() for _ in range(npoly)], dtype=f64),
                ofric=torch.tensor([0.2 + 0.6 * r() for _ in range(no)], dtype=f64))


def _oracle(sc, eps=0.1):
    """the scene's contact list in the reference's formulation (OracleHullWorld's pair walk)"""
    from lcp_physics_b200.world import polygon_centroid
    hv = torch.cat([sc["polys"], sc["obst"]])
    cen = polygon_centroid(hv)
    nh, nc = hv.shape[0], sc["pos"].shape[0]
    hp = torch.cat([torch.zeros(nh, 1, dtype=f64), cen], 1)
    z = lambda n: torch.zeros(n, dtype=f64)
    o = OracleHullWorld(sc["pos"], sc["rad"], torch.zeros(nc, 3), torch.ones(nc), z(nc), z(nc) + 0.5,
                        [v - c for v, c in zip(hv, cen)], hp, torch.zeros(nh, 3), torch.ones(nh), torch.ones(nh),
                        torch.cat([sc["pfric"], sc["ofric"]]), z(nh), [False] * nh, n_static=sc["obst"].shape[0],
                        eps=eps)
    return o


def polygon_walk(scs, dtype, cap, geometry=True, eps=0.1):
    """lcpb200_contacts with feat (the polygon walk) on a batch of scenes of equal shapes"""
    from lcp_physics_b200 import _lib
    from lcp_physics_b200.world import polygon_centroid
    lib = _lib.load()
    B = len(scs)
    st = lambda k: torch.stack([s[k] for s in scs]).to("cuda", dtype).contiguous()
    pos, rad, pv, ov = st("pos"), st("rad"), st("polys"), st("obst")
    nb, npoly, no = pos.shape[1], pv.shape[1], ov.shape[1]
    # centroids in float64 (the shoelace sums of a thin hull cancel badly in float32), then rounded to dtype
    cen = lambda k: polygon_centroid(torch.stack([s[k] for s in scs]).to("cuda", f64)).to(dtype).contiguous()
    pcen, oref = cen("polys"), cen("obst")
    fr, rs = torch.full((B, nb), 0.5, dtype=dtype, device="cuda"), torch.zeros(B, nb, dtype=dtype, device="cuda")
    pfr, ofr = st("pfric"), st("ofric")
    prs, ors = torch.zeros_like(pfr), torch.zeros_like(ofr)
    i32 = lambda *s: torch.empty(*s, dtype=torch.int32, device="cuda")
    b1, b2, feat, counts = i32(B, cap), i32(B, cap), i32(B, cap), i32(B)
    new = lambda *s: torch.empty(B, cap, *s, dtype=dtype, device="cuda")
    geo = [new(2), new(2), new(2), new(), new(), new()] if geometry else [None] * 6
    _lib.check(lib.lcpb200_contacts(
        _lib.dtype_code(dtype), B, nb, npoly, no, 6, cap, eps,
        *[_lib.ptr(t) for t in (pos, rad, fr, rs, pv, pcen, pfr, prs, ov, oref, ofr, ors, b1, b2, counts, feat)],
        *[_lib.ptr(t) for t in geo], None, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    return dict(b1=b1, b2=b2, feat=feat, counts=counts, geo=geo, pv=pv, pcen=pcen, ov=ov, oref=oref, pfr=pfr, ofr=ofr,
                pos=pos, rad=rad, fr=fr, rs=rs, prs=prs, ors=ors)


# ---------------------------------------------------------------------------------------------------- contact lists
@pytest.mark.parametrize("dtype", [f64, torch.float32])
@pytest.mark.parametrize("sizes", [(3, 8, 2, 60.0), (10, 36, 4, 140.0)])   # the second: 1 300+ pairs, 2 chunks
def test_polygon_walk_matches_polygon_oracle(sizes, dtype):
    """float32: the scenes every decision of which (rule thresholds, SAT / support / incident-edge ties, clip signs)
    clears 1e-5 x spread in the float64 restatement of the walk (tests/contact_ref.py) on the float32-rounded inputs;
    their lists equal the oracle's and their geometry is within 2e-5 x spread"""
    from tests import contact_ref as cr
    nc, npoly, no, spread = sizes
    nscenes = 4 if dtype == f64 else 8
    scs = [random_scene(100 + s, nc, npoly, no, spread) for s in range(nscenes)]
    res = polygon_walk(scs, dtype, cap=1024)
    nb, nd = nc, nc + npoly
    seen_two = seen_one = 0
    tol, compared = (1e-12 if dtype == f64 else 2e-5) * spread, 0
    for s, sc in enumerate(scs):
        if dtype != f64:
            rs = cr.make_scene(sc["pos"].numpy(), sc["rad"].numpy(), sc["polys"].numpy(), sc["obst"].numpy(), nv=6)
            if cr.scene_contacts(cr.rounded(rs, dtype), 0.1)["margin"] <= 1e-5 * spread:
                continue
        compared += 1
        orc = _oracle(sc)
        n = int(res["counts"][s])
        assert n == len(orc.contacts), (s, n, len(orc.contacts))
        assert min((min(m) for m in orc.margins), default=1.0) > 1e-9             # no tie in the random scenes
        b1, b2 = res["b1"][s, :n].tolist(), res["b2"][s, :n].tolist()
        assert [(c[4], c[5]) for c in orc.contacts] == list(zip(b1, b2)), s
        normal, p1, p2, pen, mu, _ = [t[s, :n].cpu().double() for t in res["geo"]]
        for c, (nrm, q1, q2, pn, i, j) in enumerate(orc.contacts):
            for a, b in ((normal[c], nrm), (p1[c], q1), (p2[c], q2)):      # relative to the coordinates
                assert float((a - b).abs().max()) < tol, (s, c, i, j)
            assert abs(float(pen[c]) - float(pn)) < tol
        pairs = list(zip(b1, b2))
        hh = [p for p in pairs if p[0] >= nb]
        seen_two += sum(1 for p in set(hh) if pairs.count(p) == 2)
        seen_one += sum(1 for p in set(hh) if pairs.count(p) == 1)
        assert all((f >= 0) == (i >= nb) for f, i in zip(res["feat"][s, :n].tolist(), b1))
        assert any(j >= nd for j in b2)                                            # one-body contacts
    assert compared >= 3
    assert seen_two > 0 and seen_one > 0                                           # 1- and 2-point manifolds


@pytest.mark.parametrize("dtype", [f64, torch.float32])
def test_polygon_walk_torch_geometry_from_features_matches_kernel(dtype):
    """The torch (graph) geometry BatchedWorld builds from feat equals the kernel's geometry."""
    from lcp_physics_b200.world import BatchedWorld
    scs = [random_scene(200 + s, 3, 8, 2, 60.0) for s in range(8)]
    res = polygon_walk(scs, dtype, cap=256)
    w = object.__new__(BatchedWorld)                                               # the torch mirror needs only these
    w.nb, w.np, w.no, w.nv = 3, 8, 2, 6
    w.p = torch.cat([torch.zeros(8, 11, 1, dtype=dtype, device="cuda"),
                     torch.cat([res["pos"], res["pcen"]], 1)], 2)
    w.rad, w.fric_coeff, w.restitution = res["rad"], res["fr"], res["rs"]
    w.pfric, w.prest, w.ov, w.oref, w.ofric, w.orest = res["pfr"], res["prs"], res["ov"], res["oref"], res["ofr"], res["ors"]
    got = w._geometry_torch(res["b1"], res["b2"], res["feat"], res["pv"])
    tol = 1e-12 if dtype == f64 else 2e-3
    for s in range(8):
        n = int(res["counts"][s])
        for a, b in zip(got, res["geo"]):
            scale = max(1.0, float(b[s, :n].abs().max())) if n else 1.0
            assert float((a[s, :n] - b[s, :n]).abs().max()) <= tol * scale


def test_polygon_walk_without_polygons_equals_circle_walk():
    """np == 0 through the polygon walk (lcpb200_contacts with feat) selects the same pairs as the circle walk
    (lcpb200_contacts without feat)."""
    from lcp_physics_b200 import _lib
    scs = [random_scene(300 + s, 12, 0, 3, 80.0) for s in range(4)]
    res = polygon_walk(scs, f64, cap=256)
    lib = _lib.load()
    B, cap = 4, 256
    i32 = lambda *s: torch.empty(*s, dtype=torch.int32, device="cuda")
    b1, b2, counts = i32(B, cap), i32(B, cap), i32(B)
    _lib.check(lib.lcpb200_contacts(_lib.dtype_code(f64), B, 12, 0, 3, 6, cap, 0.1,
                                    *[_lib.ptr(t) for t in (res["pos"], res["rad"], None, None, None, None, None, None,
                                                            res["ov"], res["oref"], None, None, b1, b2, counts)],
                                    None, None, None, None, None, None, None, None,
                                    ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    assert torch.equal(counts, res["counts"]) and torch.equal(b1, res["b1"]) and torch.equal(b2, res["b2"])
    assert bool((res["feat"] == -1).all())


# ---------------------------------------------------------------------------------------------------- trajectories
def golden_world(z, scene, post_stab, dtype=f64, **kw):
    from lcp_physics_b200.world import BatchedWorld
    g = lambda k: torch.from_numpy(z["%s_%s" % (scene, k)])
    ns = int(z[scene + "_nstatic"])
    hv, hp = g("hull_verts"), g("hull_p")                                           # [B, nh, V, 2], [B, nh, 3]
    wv = hv + hp[:, :, None, 1:]                                                   # world frame
    nd = hv.shape[1] - ns
    nc = z[scene + "_pos"].shape[1]
    return BatchedWorld(g("pos").reshape(hv.shape[0], nc, 2).to(dtype), g("rad").reshape(hv.shape[0], nc), vel=g("vel").reshape(hv.shape[0], nc, 3), mass=g("mass").reshape(hv.shape[0], nc),
                        restitution=g("rest"), fric_coeff=g("fric"), gravity=100.0, dt=1.0 / 30, post_stab=post_stab,
                        polygons=wv[:, :nd], poly_rot=hp[:, :nd, 0], poly_vel=g("hull_vel")[:, :nd],
                        poly_mass=g("hull_mass")[:, :nd], poly_fric=g("hull_fric")[:, :nd],
                        poly_rest=g("hull_rest")[:, :nd], obstacles=wv[:, nd:], obstacle_fric=g("hull_fric")[:, nd:],
                        obstacle_rest=g("hull_rest")[:, nd:], device="cuda", **kw), nc + nd


@pytest.mark.parametrize("post_stab", [False, True])
@pytest.mark.parametrize("scene", ["slide", "stack"])
def test_batched_world_with_polygons_reproduces_reference(scene, post_stab):
    z = np.load(GOLDEN)
    w, nd = golden_world(z, scene, post_stab)
    tag = "%s_%s_" % (scene, "ps" if post_stab else "nops")
    worst = 0.0
    for k in range(z[tag + "nc"].shape[0]):
        w.step()
        assert w.counts.cpu().tolist() == z[tag + "nc"][k].tolist(), k
        assert np.abs(w.t.cpu().numpy() - z[tag + "t"][k]).max() < 1e-12, k         # same dt-halving history
        worst = max(worst, float(np.abs(w.p.cpu().numpy() - z[tag + "p"][k][:, :nd]).max()))
    assert worst < 1e-6, worst


def test_fp32_slide_rollout_agrees_with_fp64():
    z = np.load(GOLDEN)
    w64, nd = golden_world(z, "slide", False)
    w32, _ = golden_world(z, "slide", False, dtype=torch.float32)
    assert w32.dtype == torch.float32
    for _ in range(20):
        w64.step()
        w32.step()
    d = (w32.p.double() - w64.p).abs()
    assert float(d[..., 1:].max()) < 1e-2 and float(d[..., 0].max()) < 1e-3, (float(d[..., 1:].max()),
                                                                            float(d[..., 0].max()))


# ---------------------------------------------------------------------------------------------------- large scene
def test_large_mixed_bin_matches_polygon_oracle():
    """24 boxes, 6 hulls and 20 circles (3 * 50 = 150 > 128: banded kernel) in a bin of 3 obstacles."""
    from lcp_physics_b200.world import BatchedWorld, polygon_centroid, rect_vertices
    g = torch.Generator().manual_seed(7)
    r = lambda: float(torch.rand(1, generator=g))
    base = lambda row: 500.0 - 20.06 * row - 0.03                 # bottom of the objects of each row, 0.06 apart
    polys = []
    for k in range(30):                                            # 6 columns x 5 rows
        cx, row = 130.0 + 42.0 * (k % 6), k // 6
        if k % 5 == 4:
            v = torch.tensor(_hull(cx, 0.0, 9.5, 5, r(), g), dtype=f64)
            v[:, 1] += base(row) - v[:, 1].max()
            v = v.tolist()
        else:
            v = rect_vertices([cx, base(row) - 10.0], [38.0, 20.0], 0.002 * (r() - 0.5)).tolist()
            v = v + [v[3]] * 2
        polys.append(v)
    pv = torch.tensor(polys, dtype=f64)
    pos = torch.tensor([[120.0 + 12.0 * k + 0.5 * r(), base(4) - 20.0 - 5.5 - 0.03 - 0.04 * r()] for k in range(20)],
                       dtype=f64)                                  # on the top row
    obst = torch.stack([rect_vertices([300.0, 510.0], [400.0, 20.0]), rect_vertices([90.0, 400.0], [20.0, 250.0]),
                        rect_vertices([510.0, 400.0], [20.0, 250.0])])
    obst = torch.cat([obst, obst[:, 3:].expand(-1, 2, -1)], 1)
    w = BatchedWorld(pos.unsqueeze(0), 5.5, gravity=100.0, dt=1.0 / 30, polygons=pv.unsqueeze(0), obstacles=obst,
                     obstacle_fric=0.6, obstacle_rest=0.3, restitution=0.3, fric_coeff=0.5, poly_fric=0.5,
                     poly_rest=0.3, device="cuda")
    assert w.large
    hv = torch.cat([pv, obst])
    cen = polygon_centroid(hv)
    nh = hv.shape[0]
    orc = OracleHullWorld(pos, torch.full((20,), 5.5), torch.zeros(20, 3), torch.ones(20), torch.full((20,), 0.3),
                          torch.full((20,), 0.5), [v - c for v, c in zip(hv, cen)],
                          torch.cat([torch.zeros(nh, 1, dtype=f64), cen], 1), torch.zeros(nh, 3),
                          torch.ones(nh), w.inertia[0, 20:].cpu().tolist() + [1.0] * 3,
                          [0.5] * 30 + [0.6] * 3, [0.3] * 30 + [0.3] * 3, [False] * nh, n_static=3)
    assert int(w.counts[0]) == len(orc.contacts)
    for k in range(3):
        w.step()
        orc.step()
        assert int(w.counts[0]) == len(orc.contacts), k
        err = float((w.p[0].cpu() - orc.p[:50]).abs().max())
        assert err < 1e-6, (k, err)


# ---------------------------------------------------------------------------------------------------- gradients
def test_sliding_box_rollout_gradients_match_central_differences():
    """A Rect sliding on a pinned floor (a 2-point manifold from step 0): d(final x, rot) / d(initial velocity,
    friction, mass, dims) through 6 steps with exact_adjoint=True, against central differences (every solve
    converged below 1e-8)."""
    from lcp_physics_b200.engines import last_solve_info
    from lcp_physics_b200.world import BatchedWorld, rect_vertices
    dev = "cuda"
    floor = rect_vertices(torch.tensor([300.0, 520.0], dtype=f64, device=dev),
                          torch.tensor([600.0, 20.0], dtype=f64, device=dev)).unsqueeze(0)

    def rollout(vx, fric, mass, dims):
        ctr = torch.stack([torch.tensor(200.0, dtype=f64, device=dev), 510.0 - dims[1] / 2 - 0.03])
        verts = rect_vertices(ctr, dims, torch.tensor(0.001, dtype=f64, device=dev))
        vel = torch.stack([torch.zeros_like(vx), vx, torch.zeros_like(vx)]).reshape(1, 1, 3)
        w = BatchedWorld(torch.zeros(1, 0, 2, dtype=f64, device=dev), 1.0, gravity=100.0, dt=1.0 / 60,
                         polygons=verts.unsqueeze(0), poly_vel=vel, poly_mass=mass.reshape(1, 1),
                         poly_fric=fric.reshape(1, 1), poly_rest=0.0, obstacles=floor, obstacle_fric=0.2,
                         obstacle_rest=0.0, exact_adjoint=True, device=dev, tol=1e-4)
        for _ in range(6):
            w.step()
            info = last_solve_info()
            assert bool((info["status"] == 2).all()) and float(info["resid"].max()) < 1e-8
        return w.p[0, 0, 1] + 10.0 * w.p[0, 0, 0]

    x0 = [torch.tensor(v, dtype=f64, device=dev) for v in (30.0, 0.1, 1.5)]
    d0 = torch.tensor([40.0, 20.0], dtype=f64, device=dev)
    leaves = [t.clone().requires_grad_(True) for t in x0 + [d0]]
    y = rollout(*leaves)
    grads = torch.autograd.grad(y, leaves)
    h = 1e-5
    with torch.no_grad():
        for k in range(4):
            for comp in range(leaves[k].numel()):
                plus = [t.detach().clone() for t in leaves]
                minus = [t.detach().clone() for t in leaves]
                plus[k].view(-1)[comp] += h
                minus[k].view(-1)[comp] -= h
                fd = float((rollout(*plus) - rollout(*minus)) / (2 * h))
                g = float(grads[k].reshape(-1)[comp])
                assert abs(g - fd) <= 1e-3 * max(abs(fd), 1e-2), (k, comp, g, fd)


def test_polygon_world_api_errors():
    from lcp_physics_b200.world import BatchedWorld, rect_vertices
    sq = rect_vertices([0.0, 0.0], [10.0, 10.0])
    with pytest.raises(ValueError, match="orientation"):
        BatchedWorld(torch.zeros(1, 0, 2, dtype=f64), 1.0, polygons=sq.flip(0).unsqueeze(0), device="cuda")
    w = BatchedWorld(torch.zeros(1, 0, 2, dtype=f64), 1.0, polygons=sq.unsqueeze(0), device="cuda")
    assert w.nd == 1 and w.get_p().shape == (1, 3) and w.mass.shape == (1, 1)
    assert abs(float(w.inertia[0, 0]) - 200.0 / 12) < 1e-12                       # Rect: m (w^2 + h^2) / 12
    with pytest.raises(NotImplementedError):
        w.find_contacts_torch()
    w.step()
    assert float(w.p[0, 0, 2]) > 0                                                # falls under gravity
