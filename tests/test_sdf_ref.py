"""CPU: the signed-distance rule of lcpb200_signed_distance on hand-worked cases, for the brute-force reference
(tests/sdf_ref.py) and the torch mirror that BatchedWorld.signed_distance differentiates through
(BatchedWorld._sdf_torch, called here on a stand-in for the world's state); the mirror's gradients against finite
differences; the pixel centres of BatchedWorld.render."""
import math
import types

import pytest
import torch

from tests.sdf_ref import sdf_ref

f64 = torch.float64
R2 = math.sqrt(0.5)


def box(cx, cy, w, h):
    """axis-aligned box, positive orientation: (x1, y1), (x0, y1), (x0, y0), (x1, y0) -- edges top, left, bottom, right"""
    x0, x1, y0, y1 = cx - w / 2, cx + w / 2, cy - h / 2, cy + h / 2
    return [[x1, y1], [x0, y1], [x0, y0], [x1, y0]]


def stand_in(c, pv, ov):
    """the attributes of BatchedWorld that _sdf_torch reads"""
    from lcp_physics_b200.world import polygon_centroid
    nb, np_ = c.shape[1], 0 if pv is None else pv.shape[1]
    p = torch.cat([torch.zeros(1, nb, 1, dtype=f64), c[..., :2]], 2)
    if np_:
        p = torch.cat([p, torch.cat([torch.zeros(1, np_, 1, dtype=f64), polygon_centroid(pv)], 2)], 1)
    nv = max(0 if pv is None else pv.shape[2], 0 if ov is None else ov.shape[2])
    return types.SimpleNamespace(nb=nb, np=np_, no=0 if ov is None else ov.shape[1], nv=nv, p=p, rad=c[..., 2], ov=ov)


def mirror(c, pv, ov, x, body, feat, max_dist):
    from lcp_physics_b200.world import BatchedWorld
    return BatchedWorld._sdf_torch(stand_in(c, pv, ov), x, body, feat, max_dist, pv)


def query(circles=(), polys=(), obst=(), points=(), max_dist=100.0, active=None):
    """one scene: circles [(x, y, r)], polygons / obstacles [[V, 2]] (equal V), points [(x, y)]; checks the mirror
    against the reference and returns the reference's (sdf, body, feat, normal) as lists"""
    c = torch.tensor(circles, dtype=f64).reshape(1, -1, 3)
    pv = torch.tensor(polys, dtype=f64).reshape(1, len(polys), -1, 2) if polys else None
    ov = torch.tensor(obst, dtype=f64).reshape(1, len(obst), -1, 2) if obst else None
    x = torch.tensor(points, dtype=f64).reshape(1, -1, 2)
    act = None if active is None else torch.tensor(active).reshape(1, -1)
    sdf, body, feat, normal, _ = sdf_ref(c[..., :2], c[..., 2], pv, ov, x, max_dist, act)
    m = mirror(c, pv, ov, x, body, feat, max_dist)
    fin = torch.isfinite(x).all(2)
    assert torch.allclose(m[0][fin], sdf[fin], rtol=1e-15, atol=1e-15), (m[0], sdf)
    assert torch.allclose(m[1][fin], normal[fin], rtol=1e-15, atol=1e-15), (m[1], normal)
    return sdf[0].tolist(), body[0].tolist(), feat[0].tolist(), normal[0].tolist()


def close(a, b):
    return a == pytest.approx(b, rel=1e-15, abs=1e-15)


def test_circle_outside_inside_and_at_the_centre():
    s, b, f, n = query(circles=[(0.0, 0.0, 1.0)], points=[(3.0, 4.0), (0.5, 0.0), (0.0, 0.0)])
    assert s == [4.0, -0.5, -1.0] and b == [0, 0, 0] and f == [-1, -1, -1]
    assert close(n[0], [0.6, 0.8]) and n[1] == [1.0, 0.0] and n[2] == [0.0, 0.0]


def test_box_face_corner_inside_and_on_an_edge():
    scene = dict(polys=[box(0.0, 0.0, 2.0, 2.0)])
    s, b, f, n = query(**scene, points=[(3.0, 0.0), (2.0, 2.0), (0.5, 0.2), (1.0, 0.3), (0.0, -3.0)])
    assert b == [0] * 5
    assert s[0] == 2.0 and f[0] == 3 and n[0] == [1.0, 0.0]                       # the right face
    assert close(s[1], math.sqrt(2.0)) and f[1] == 0 and close(n[1], [R2, R2])    # corner (1, 1): edges 0 and 3 tie
    assert close(s[2], -0.5) and f[2] == 256 + 3 and n[2] == [1.0, 0.0]          # inside: the nearest face
    assert s[3] == 0.0 and f[3] == 256 + 3 and n[3] == [1.0, 0.0]                # on the right edge
    assert s[4] == 2.0 and f[4] == 2 and n[4] == [0.0, -1.0]


def test_corner_regions_report_the_first_edge():
    # each corner's region: the lower of the two edges meeting there (vertex 0 joins edges 3 and 0: edge 0)
    pts = [(2.0, 2.0), (-2.0, 2.0), (-2.0, -2.0), (2.0, -2.0)]
    s, _, f, n = query(polys=[box(0.0, 0.0, 2.0, 2.0)], points=pts)
    assert f == [0, 0, 1, 2]
    assert all(close(v, math.sqrt(2.0)) for v in s)
    assert close(n[2], [-R2, -R2])


def test_padded_polygon_equals_the_unpadded_one():
    tri = [[3.0, -1.0], [5.0, 0.0], [3.0, 1.0]]
    pts = [(0.0, 0.0), (3.5, 0.1), (4.5, 1.5), (3.0, 2.0)]
    s3, _, f3, n3 = query(polys=[tri], points=pts)
    s5, _, f5, n5 = query(polys=[tri + [[3.0, 1.0], [3.0, 1.0]]], points=pts)
    assert s3 == s5 and n3 == n5
    assert f3 == [2, 256 + 2, 1, 1]
    assert f5 == [4, 256 + 4, 1, 1]                    # the repeated vertex's zero-length edges are skipped
    assert s3[0] == 3.0 and n3[0] == [-1.0, 0.0] and close(s3[1], -0.5)


def test_reversed_orientation_obstacle():
    pts = [(3.0, 0.0), (0.5, 0.2), (2.0, 2.0)]
    sp, _, fp, np_ = query(polys=[box(0.0, 0.0, 2.0, 2.0)], points=pts)
    so, bo, fo, no = query(obst=[box(0.0, 0.0, 2.0, 2.0)[::-1]], points=pts)
    assert so == sp and no == np_ and bo == [0, 0, 0]
    assert fo == [3, 256 + 3, 2]                       # edges of the reversed list: bottom, left, top, right


def test_overlapping_bodies_min_wins():
    s, b, f, _ = query(circles=[(0.0, 0.0, 0.5)], polys=[box(0.0, 0.0, 4.0, 4.0)], points=[(0.0, 0.0), (0.1, 0.0)])
    assert b == [1, 1] and s[0] == -2.0 and f[0] == 256 + 0
    s, b, _, _ = query(circles=[(0.0, 0.0, 3.0)], polys=[box(0.0, 0.0, 2.0, 2.0)], points=[(0.5, 0.0)])
    assert (s, b) == ([-2.5], [0])


def test_exact_tie_goes_to_the_lower_index():
    s, b, _, _ = query(circles=[(-2.0, 0.0, 1.0), (2.0, 0.0, 1.0)], points=[(0.0, 0.0)])
    assert (s, b) == ([1.0], [0])
    s, b, _, _ = query(circles=[(2.0, 0.0, 1.0), (-2.0, 0.0, 1.0)], points=[(0.0, 0.0)])
    assert (s, b) == ([1.0], [0])
    # a circle (body 0) and a box (body 1) both at distance 1
    s, b, f, _ = query(circles=[(2.0, 0.0, 1.0)], polys=[box(-2.0, 0.0, 2.0, 2.0)], points=[(0.0, 0.0)])
    assert (s, b, f) == ([1.0], [0], [-1])


def test_max_dist_inactive_and_non_finite():
    scene = dict(circles=[(10.0, 0.0, 1.0)])
    assert query(**scene, points=[(0.0, 0.0)], max_dist=5.0) == ([5.0], [-1], [-1], [[0.0, 0.0]])
    assert query(**scene, points=[(0.0, 0.0)], max_dist=9.0)[:3] == ([9.0], [0], [-1])     # sdf <= max_dist
    s, b, _, _ = query(circles=[(3.0, 0.0, 1.0), (8.0, 0.0, 1.0)], points=[(0.0, 0.0)], active=[False, True])
    assert (s, b) == ([7.0], [1])
    s, b, f, n = query(**scene, points=[(math.nan, 0.0), (0.0, math.inf)], max_dist=50.0)
    assert (s, b, f, n) == ([50.0, 50.0], [-1, -1], [-1, -1], [[0.0, 0.0], [0.0, 0.0]])


def test_margin_sees_near_decisions():
    # 1e-6 off the vertex region's boundary, 1e-6 inside the face, 1e-6 from a second body
    c = torch.zeros(1, 0, 2, dtype=f64)
    pv = torch.tensor([box(0.0, 0.0, 2.0, 2.0)], dtype=f64).unsqueeze(0)
    x = torch.tensor([[[2.0, 1.0 - 1e-6], [1.0 - 1e-6, 0.0], [3.0, 0.0]]], dtype=f64)
    m = sdf_ref(c, torch.zeros(1, 0, dtype=f64), pv, None, x, 50.0)[4][0]
    assert float(m[0]) < 1e-5 and float(m[1]) < 1e-5 and float(m[2]) > 0.2
    m = sdf_ref(torch.tensor([[[0.0, 0.0], [4.0 + 1e-6, 0.0]]], dtype=f64), torch.ones(1, 2, dtype=f64), None, None,
                torch.tensor([[[2.0, 0.0]]], dtype=f64), 50.0)[4]
    assert float(m) < 1e-5


def test_mirror_gradients_against_central_differences():
    """d(sdf, normal) / d(points, circle pos / radius, polygon and obstacle vertices) of the mirror, the choices
    (body, feat) held at the reference's; finite at a circle's centre"""
    g = torch.Generator().manual_seed(3)
    c = torch.tensor([[[6.0, 1.0, 1.5], [2.0, 7.0, 1.0]]], dtype=f64)
    pv = torch.tensor([box(-6.0, 1.0, 2.0, 3.0)], dtype=f64).unsqueeze(0)
    ov = torch.tensor([[[1.0, -6.0], [4.0, -5.0], [-2.0, -4.5], [-3.0, -6.5]][::-1]], dtype=f64).unsqueeze(0)
    x = torch.cat([20 * torch.rand(1, 40, 2, generator=g, dtype=f64) - 10,
                   torch.tensor([[[6.3, 1.2], [-6.2, 1.4], [0.5, -5.3]]], dtype=f64)], 1)   # inside each kind
    leaves = [x.requires_grad_(), c.requires_grad_(), pv.requires_grad_(), ov.requires_grad_()]
    with torch.no_grad():
        _, body, feat, _, margin = sdf_ref(c[..., :2], c[..., 2], pv, ov, x, 3.0)
    robust = margin > 1e-3
    assert set(body[0].tolist()) == {-1, 0, 1, 2, 3} and int(robust.sum()) >= 35, (body, int(robust.sum()))
    assert bool((feat >= 256).any()) and bool(((feat >= 0) & (feat < 256)).any())

    def f(x, c, pv, ov):
        s, n = mirror(c, pv, ov, x, body, feat, 3.0)
        return torch.cat([s.unsqueeze(2), n], 2) * robust.unsqueeze(2)

    wt = torch.rand(1, 43, 3, generator=g, dtype=f64)
    grads = torch.autograd.grad((f(*leaves) * wt).sum(), leaves)
    h = 1e-6
    for k, (lf, gx) in enumerate(zip(leaves, grads)):
        flat = lf.detach().reshape(-1)
        fd = torch.empty_like(flat)
        for i in range(flat.numel()):
            args = [l.detach() for l in leaves]
            xp, xm = flat.clone(), flat.clone()
            xp[i] += h
            xm[i] -= h
            args[k] = xp.reshape(lf.shape)
            yp = (f(*args) * wt).sum()
            args[k] = xm.reshape(lf.shape)
            ym = (f(*args) * wt).sum()
            fd[i] = (yp - ym) / (2 * h)
        scale = fd.abs().max().clamp_min(1.0)
        assert float((gx.reshape(-1) - fd).abs().max() / scale) < 1e-6, k
    # at a circle's centre: sdf -r, a zero normal, finite gradients in both modes
    xc = torch.tensor([[[6.0, 1.0]]], dtype=f64, requires_grad=True)
    s, n = mirror(c.detach(), None, None, xc, torch.zeros(1, 1, dtype=torch.int64),
                  torch.full((1, 1), -1, dtype=torch.int64), 9.0)
    assert float(s) == -1.5 and n.abs().sum() == 0
    gx, = torch.autograd.grad(s.sum() + n.sum(), xc)
    assert bool(torch.isfinite(gx).all())
    import torch.autograd.forward_ad as fwAD
    with fwAD.dual_level():
        s, n = mirror(c.detach(), None, None, fwAD.make_dual(xc.detach(), torch.ones_like(xc)),
                      torch.zeros(1, 1, dtype=torch.int64), torch.full((1, 1), -1, dtype=torch.int64), 9.0)
        assert bool(torch.isfinite(fwAD.unpack_dual(s).tangent).all())
        assert bool(torch.isfinite(fwAD.unpack_dual(n).tangent).all())


def test_pixel_centres():
    from lcp_physics_b200.world import pixel_centres
    lo, hi = torch.tensor([0.0, 0.0], dtype=f64), torch.tensor([3.0, 2.0], dtype=f64)
    pc = pixel_centres(2, 3, lo, hi)
    assert pc.tolist() == [[0.5, 0.5], [1.5, 0.5], [2.5, 0.5], [0.5, 1.5], [1.5, 1.5], [2.5, 1.5]]   # row i grows with y
    lo2 = torch.tensor([[0.0, 0.0], [-1.0, 10.0]], dtype=f64, requires_grad=True)
    hi2 = torch.tensor([[3.0, 2.0], [1.0, 14.0]], dtype=f64)
    pc2 = pixel_centres(2, 3, lo2, hi2)
    assert pc2.shape == (2, 6, 2) and torch.equal(pc2[0].detach(), pc)
    i, j = 1, 2
    assert pc2[1, i * 3 + j].tolist() == [-1.0 + (j + 0.5) * 2.0 / 3, 10.0 + (i + 0.5) * 4.0 / 2]
    g, = torch.autograd.grad(pc2[1, :, 0].sum(), lo2)                  # x = lo_x + (j + 1/2)(hi_x - lo_x) / W
    assert g[1].tolist() == pytest.approx([6 * (1 - (0.5 + 1.5 + 2.5) / 3 / 3), 0.0])
