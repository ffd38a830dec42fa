"""CPU: the shape-cast and sweep rule of lcpb200_shapecast on hand-worked cases, for the brute-force reference
(tests/sweep_ref.py) and the torch mirrors that BatchedWorld.shapecast / sweep differentiate through
(BatchedWorld._ray_torch with an inflation radius, and BatchedWorld._sweep_torch, called here on a stand-in for the
world's state with the kernel's choices worked out by hand); the mirrors' gradients against central differences."""
import math
import types

import pytest
import torch

from tests.sweep_ref import shapecast_ref, sweep_ref
from tests.test_sdf_ref import box

f64 = torch.float64


def feat(tf, vtx=0, src_b=0):
    """the packing of lcpb200_shapecast's feat"""
    return tf | vtx << 9 | src_b << 17


def stand_in(c, pv, ov):
    """the attributes of BatchedWorld that _sweep_torch and _ray_torch read"""
    from lcp_physics_b200.world import BatchedWorld
    nb = c.shape[1]
    np_ = 0 if pv is None else pv.shape[1]
    p = torch.cat([torch.zeros(1, nb, 1, dtype=f64), c[..., :2]], 2)
    if np_:
        p = torch.cat([p, torch.zeros(1, np_, 3, dtype=f64)], 1)
    nv = max(0 if pv is None else pv.shape[2], 0 if ov is None else ov.shape[2])
    w = types.SimpleNamespace(nb=nb, np=np_, no=0 if ov is None else ov.shape[1], nv=nv, p=p, rad=c[..., 2], ov=ov,
                              dtype=f64, device=torch.device("cpu"))
    w._ray_torch = lambda *a: BatchedWorld._ray_torch(w, *a)
    return w


def scene(circles=(), polys=(), obst=()):
    c = torch.tensor(circles, dtype=f64).reshape(1, -1, 3)
    pv = torch.tensor(polys, dtype=f64).reshape(1, len(polys), -1, 2) if polys else None
    ov = torch.tensor(obst, dtype=f64).reshape(1, len(obst), -1, 2) if obst else None
    return c, pv, ov


def cast(sc, queries, feats, max_dist=50.0):
    """queries [(ox, oy, ux, uy, r)] (u of unit length): the reference, and the mirror on the hand-worked feats (bits
    0-8, None for a miss) of the reference's bodies; returns the reference's (dist, body, normal, margin) as lists and
    the mirror's (dist, normal, point)"""
    from lcp_physics_b200.world import BatchedWorld
    c, pv, ov = sc
    q = torch.tensor(queries, dtype=f64).reshape(1, -1, 5)
    o, u, r = q[..., :2], q[..., 2:4], q[..., 4]
    d, body, n, margin = shapecast_ref(c[..., :2], c[..., 2], pv, ov, o, u, r, max_dist)
    fs = torch.tensor([[-1 if f is None else f for f in feats]])
    assert torch.equal(body >= 0, fs >= 0)
    t, m = BatchedWorld._ray_torch(stand_in(c, pv, ov), o, u, body, fs, max_dist, pv, r)
    hit = (body >= 0).unsqueeze(2)
    point = torch.where(hit, o + t.unsqueeze(2) * u - r.unsqueeze(2) * m, torch.zeros_like(o))
    robust = margin > 1e-6
    assert torch.allclose(t[robust], d[robust], rtol=1e-12, atol=1e-12), (t, d)
    assert torch.allclose(m[robust], n[robust], rtol=1e-12, atol=1e-12), (m, n)
    return d[0].tolist(), body[0].tolist(), n[0].tolist(), margin[0].tolist(), t[0].tolist(), m[0].tolist(), \
        point[0].tolist()


def sweep(sc, queries, feats):
    """queries [(body, dx, dy)]: the reference, and the mirror on the hand-worked feats (None for a miss); returns the
    reference's (frac, body, normal, margin) and the mirror's (frac, normal, point) as lists"""
    from lcp_physics_b200.world import BatchedWorld
    c, pv, ov = sc
    bq = torch.tensor([[q[0] for q in queries]])
    disp = torch.tensor([[q[1:] for q in queries]], dtype=f64)
    fr, body, n, margin = sweep_ref(c[..., :2], c[..., 2], pv, ov, bq, disp)
    fs = torch.tensor([[-1 if f is None else f for f in feats]])
    assert torch.equal(body >= 0, fs >= 0)
    L = disp.norm(dim=2)
    Ls = torch.where(L > 0, L, torch.ones_like(L))
    mf, _, mn, mp = BatchedWorld._sweep_torch(stand_in(c, pv, ov), bq, body, fs, disp / Ls.unsqueeze(2), Ls, pv)
    robust = margin > 1e-6
    assert torch.allclose(mf[robust], fr[robust], rtol=1e-12, atol=1e-12), (mf, fr)
    assert torch.allclose(mn[robust], n[robust], rtol=1e-12, atol=1e-12), (mn, n)
    return fr[0].tolist(), body[0].tolist(), n[0].tolist(), margin[0].tolist(), mf[0].tolist(), mn[0].tolist(), \
        mp[0].tolist()


def approx(v):
    """pytest.approx of a number or a (nested) list, compared flattened"""
    flat = lambda x: [z for y in x for z in flat(y)] if isinstance(x, list) else [x]
    a = pytest.approx(flat(v), rel=1e-12, abs=1e-12)
    return _Approx(a, flat)


class _Approx:
    """equal to a (nested) list whose flattened entries approx a holds"""

    def __init__(self, a, flat):
        self.a, self.flat = a, flat

    def __eq__(self, other):
        return self.flat(other) == self.a


def test_disk_onto_a_box_face_and_corner():
    sc = scene(polys=[box(0.0, 0.0, 2.0, 2.0)])
    # face: the disk's centre stops on the offset line x = -1.5; corner: |(x, 1.3) - (-1, 1)| = 0.5 at x = -1.4
    d, body, n, _, t, m, pt = cast(sc, [(-5.0, 0.0, 1.0, 0.0, 0.5), (-5.0, 1.3, 1.0, 0.0, 0.5)], [1, 256 + 1])
    assert body == [0, 0]
    assert d[0] == approx(3.5) and n[0] == approx([-1.0, 0.0]) and pt[0] == approx([-1.0, 0.0])
    assert d[1] == approx(3.6) and n[1] == approx([-0.8, 0.6]) and pt[1] == approx([-1.0, 1.0])
    assert m[1] == approx([-0.8, 0.6]) and t[1] == approx(3.6)
    # radius 0 is a ray cast: the left face at x = -1
    d, body, _, _, _, _, _ = cast(sc, [(-5.0, 0.25, 1.0, 0.0, 0.0)], [1])
    assert d == approx([4.0]) and body == [0]


def test_grazing_circle_has_no_margin():
    sc = scene(circles=[(0.0, 0.0, 1.0)])
    d, body, n, margin, t, m, _ = cast(sc, [(-5.0, 2.0, 1.0, 0.0, 1.0)], [0])
    assert body == [0] and d[0] == pytest.approx(5.0, abs=1e-6) and margin[0] < 1e-6
    assert t == [5.0] and m == [[0.0, 1.0]]                    # the mirror: disc = 0, the tangent point


def test_squares_face_to_face_and_corner_to_face():
    diamond = [[1.0, 0.0], [0.0, 1.0], [-1.0, 0.0], [0.0, -1.0]]
    sc = scene(polys=[box(0.0, 0.0, 2.0, 2.0), box(4.0, 0.0, 2.0, 2.0)])
    # A's vertex 0 (1, 1) reaches B's left face (edge 1) after 2 of 5: the first of A's two vertices on that face
    fr, body, n, _, mf, mn, mp = sweep(sc, [(0, 5.0, 0.0)], [feat(1, 0, 0)])
    assert fr == approx([0.4]) and body == [1] and n == approx([[1.0, 0.0]]) and mp == approx([[3.0, 1.0]])
    sc = scene(polys=[diamond, box(4.0, 0.0, 2.0, 2.0)])
    # corner to face: the diamond's vertex 0 meets x = 3 after 2 of 4
    fr, body, n, _, _, mn, mp = sweep(sc, [(0, 4.0, 0.0)], [feat(1, 0, 0)])
    assert fr == approx([0.5]) and body == [1] and n == approx([[1.0, 0.0]]) and mp == approx([[3.0, 0.0]])
    # the box moving onto the diamond: the diamond's vertex 0, cast backwards, is the source (bit 17)
    fr, body, n, _, _, mn, mp = sweep(sc, [(1, -4.0, 0.0)], [feat(1, 0, 1)])
    assert fr == approx([0.5]) and body == [0] and n == approx([[-1.0, 0.0]]) and mp == approx([[1.0, 0.0]])


def test_touching_overlapping_and_limit():
    sc = scene(circles=[(0.0, 0.0, 1.0), (2.0, 0.0, 1.0), (0.0, 1.5, 1.0)], polys=[box(10.0, 0.0, 2.0, 2.0)])
    # body 0 touches 1 and overlaps 2: approaching 1 reads 0, leaving it (or moving into 2 only) misses
    fr, body, n, _, mf, mn, mp = sweep(sc, [(0, 1.0, 0.0), (0, -1.0, 0.0), (0, 0.0, 1.0)], [feat(0), None, None])
    assert fr == [0.0, 1.0, 1.0] and body == [1, -1, -1] and mn[0] == [1.0, 0.0] and mp[0] == [1.0, 0.0]
    assert mf == [0.0, 1.0, 1.0] and mn[1] == [0.0, 0.0] == mp[1]
    # the limit exactly at the hit: body 1's circle reaches the box's left face (x = 9) after exactly 6
    fr, body, _, margin, mf, _, mp = sweep(sc, [(1, 6.0, 0.0)], [feat(1)])
    assert body == [3] and fr == approx([1.0]) and mf == [1.0] and margin[0] < 1e-6 and mp == [[9.0, 0.0]]
    # a box sweeping onto a circle: the circle, cast backwards against the box, is the source
    fr, body, n, _, _, mn, mp = sweep(sc, [(3, -10.0, 0.0)], [feat(1, 0, 1)])
    assert body == [1] and fr == approx([0.6]) and n == approx([[-1.0, 0.0]]) and mp == approx([[3.0, 0.0]])


def test_padded_polygons_and_reversed_obstacles():
    sq = box(0.0, 0.0, 2.0, 2.0)
    a = cast(scene(polys=[sq + [sq[-1]]]), [(-5.0, 0.0, 1.0, 0.0, 0.5), (-5.0, 1.3, 1.0, 0.0, 0.5)], [1, 257])
    b = cast(scene(obst=[sq[::-1] + [sq[0]]]), [(-5.0, 0.0, 1.0, 0.0, 0.5), (-5.0, 1.3, 1.0, 0.0, 0.5)], [1, 256 + 2])
    assert a[0] == approx(b[0]) and a[2] == approx(b[2]) and a[6] == approx(b[6])
    tri = [[3.0, -1.0], [5.0, 0.0], [3.0, 1.0]]
    # padded, either orientation: the left face x = 3 is edge 4 (edges 2 and 3 have zero length)
    s1 = sweep(scene(polys=[sq + [sq[-1]], tri + [tri[-1]] * 2]), [(0, 4.0, 0.0)], [feat(4, 0, 0)])
    s2 = sweep(scene(polys=[sq + [sq[-1]]], obst=[tri[::-1] + [tri[0]] * 2]), [(0, 4.0, 0.0)], [feat(4, 0, 0)])
    assert s1[0] == approx([0.5]) == s2[0] and s1[2] == approx([[1.0, 0.0]]) == s2[2]


def test_mirror_gradients_against_central_differences():
    """d(shape cast, sweep outputs) / d(circles, polygon and obstacle vertices, origins, directions, radii,
    displacements) of the mirrors, the choices held"""
    from lcp_physics_b200.world import BatchedWorld
    c = torch.tensor([[[6.0, 1.0, 1.5], [2.0, 7.0, 1.0]]], dtype=f64)
    pv = torch.tensor([[[-5.0, 2.0], [-7.0, 2.5], [-7.5, -0.5], [-5.5, -1.0]]], dtype=f64).unsqueeze(0)
    ov = torch.tensor([[[1.0, -6.0], [4.0, -5.0], [-2.0, -4.5], [-3.0, -6.5]][::-1]], dtype=f64).unsqueeze(0)
    o = torch.tensor([[[0.0, 1.2], [0.3, -1.0], [-1.0, 0.5]]], dtype=f64)
    ang = torch.tensor([[0.1, -1.7, 2.9]], dtype=f64)
    rq = torch.tensor([[0.7, 0.4, 0.0]], dtype=f64)
    bq = torch.tensor([[0, 1, 2, 3]])
    disp = torch.tensor([[[-4.0, -9.0], [4.0, -6.0], [9.0, -7.0], [3.0, 9.0]]], dtype=f64)
    u = torch.stack([ang.cos(), ang.sin()], 2)
    dr, br, _, mr = shapecast_ref(c[..., :2], c[..., 2], pv, ov, o, u, rq, 50.0)
    fr, bs, _, ms = sweep_ref(c[..., :2], c[..., 2], pv, ov, bq, disp)
    assert bool((br >= 0).all()) and bool((bs >= 0).all()), (br, bs)
    assert bool((mr > 1e-3).all()) and bool((ms > 1e-3).all()), (mr, ms)
    # the kernel's choices, read off the reference's contacts by hand
    # casts: circle 0, the obstacle's top face 1, the polygon's face 3; sweeps: circle 0 onto the obstacle's face 1,
    # circle 1 onto circle 0, the polygon's vertex 3 onto the obstacle's face 1, the obstacle onto circle 0, whose
    # centre (cast backwards) meets the obstacle's vertex 2
    fc = torch.tensor([[0, 1, 3]])
    fsw = torch.tensor([[feat(1), feat(0), feat(1, 3, 0), feat(256 + 2, 0, 1)]])
    w = stand_in(c, pv, ov)
    leaves = [c.clone().requires_grad_(), pv.clone().requires_grad_(), ov.clone().requires_grad_(),
              o.clone().requires_grad_(), ang.clone().requires_grad_(), rq.clone().requires_grad_(),
              disp.clone().requires_grad_()]

    def f(c_, pv_, ov_, o_, ang_, rq_, disp_):
        w.p = torch.cat([torch.cat([torch.zeros(1, 2, 1, dtype=f64), c_[..., :2]], 2), torch.zeros(1, 1, 3, dtype=f64)],
                        1)
        w.rad, w.ov = c_[..., 2], ov_
        u_ = torch.stack([ang_.cos(), ang_.sin()], 2)
        t, m = BatchedWorld._ray_torch(w, o_, u_, br, fc, 50.0, pv_, rq_)
        L = disp_.norm(dim=2)
        sw = BatchedWorld._sweep_torch(w, bq, bs, fsw, disp_ / L.unsqueeze(2), L, pv_)
        return torch.cat([t.reshape(-1), m.reshape(-1), sw[0].reshape(-1), sw[2].reshape(-1), sw[3].reshape(-1)])

    y = f(*leaves)
    assert torch.allclose(y[:3], dr[0], rtol=1e-12) and torch.allclose(y[9:13], fr[0], rtol=1e-12)
    wt = torch.rand(y.shape, generator=torch.Generator().manual_seed(5), dtype=f64)
    grads = torch.autograd.grad((y * wt).sum(), leaves)
    h = 1e-6
    for k, (lf, gx) in enumerate(zip(leaves, grads)):
        flat = lf.detach().reshape(-1)
        fd = torch.empty_like(flat)
        for i in range(flat.numel()):
            args = [x.detach() for x in leaves]
            ys = []
            for sgn in (1.0, -1.0):
                xp = flat.clone()
                xp[i] += sgn * h
                args[k] = xp.reshape(lf.shape)
                ys.append((f(*args) * wt).sum())
            fd[i] = (ys[0] - ys[1]) / (2 * h)
        assert float((gx.reshape(-1) - fd).abs().max() / fd.abs().max().clamp_min(1.0)) < 1e-6, k
        assert float(gx.abs().max()) > 0, k
