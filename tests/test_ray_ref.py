"""CPU: the ray-cast rule of lcpb200_raycast on hand-worked cases, for the brute-force reference (tests/ray_ref.py) and the
torch mirror that BatchedWorld.raycast differentiates through (BatchedWorld._ray_torch, called here on a stand-in for the
world's state), and the mirror's gradients against finite differences."""
import math
import types

import pytest
import torch

from tests.ray_ref import ray_ref

f64 = torch.float64


def box(cx, cy, w, h):
    """axis-aligned box, positive orientation: (x1, y1), (x0, y1), (x0, y0), (x1, y0) -- edges top, left, bottom, right"""
    x0, x1, y0, y1 = cx - w / 2, cx + w / 2, cy - h / 2, cy + h / 2
    return [[x1, y1], [x0, y1], [x0, y0], [x1, y0]]


def cast(circles=(), polys=(), obst=(), rays=(), max_dist=100.0, active=None):
    """one scene: circles [(x, y, r)], polygons / obstacles [[V, 2]] (equal V), rays [(ox, oy, dx, dy)]"""
    c = torch.tensor(circles, dtype=f64).reshape(1, -1, 3)
    pv = torch.tensor(polys, dtype=f64).reshape(1, len(polys), -1, 2) if polys else None
    ov = torch.tensor(obst, dtype=f64).reshape(1, len(obst), -1, 2) if obst else None
    r = torch.tensor(rays, dtype=f64).reshape(1, -1, 4)
    d = r[..., 2:] / r[..., 2:].norm(dim=2, keepdim=True)
    act = None if active is None else torch.tensor(active).reshape(1, -1)
    out = ray_ref(c[..., :2], c[..., 2], pv, ov, r[..., :2], d, max_dist, act)
    t, body, feat, normal, _ = out
    mirror = mirror_cast(c, pv, ov, r[..., :2], d, body, feat, max_dist)
    assert torch.allclose(mirror[0], t, rtol=1e-15, atol=1e-15), (mirror[0], t)
    assert torch.allclose(mirror[1], normal, rtol=1e-15, atol=1e-15), (mirror[1], normal)
    return t[0].tolist(), body[0].tolist(), feat[0].tolist(), normal[0].tolist()


def stand_in(c, pv, ov):
    """the attributes of BatchedWorld that _ray_torch reads"""
    from lcp_physics_b200.world import polygon_centroid
    nb, np_ = c.shape[1], 0 if pv is None else pv.shape[1]
    p = torch.cat([torch.zeros(1, nb, 1, dtype=f64), c[..., :2]], 2)
    if np_:
        p = torch.cat([p, torch.cat([torch.zeros(1, np_, 1, dtype=f64), polygon_centroid(pv)], 2)], 1)
    nv = max(0 if pv is None else pv.shape[2], 0 if ov is None else ov.shape[2])
    return types.SimpleNamespace(nb=nb, np=np_, no=0 if ov is None else ov.shape[1], nv=nv, p=p, rad=c[..., 2], ov=ov)


def mirror_cast(c, pv, ov, o, u, body, feat, max_dist):
    from lcp_physics_b200.world import BatchedWorld
    return BatchedWorld._ray_torch(stand_in(c, pv, ov), o, u, body, feat, max_dist, pv)


def test_axis_ray_into_a_circle_and_a_box():
    t, b, f, n = cast(circles=[(5.0, 0.0, 1.0)], rays=[(0.0, 0.0, 1.0, 0.0), (0.0, 0.0, 0.0, 2.0)])
    assert (t, b, f, n) == ([4.0, 100.0], [0, -1], [-1, -1], [[-1.0, 0.0], [0.0, 0.0]])
    t, b, f, n = cast(polys=[box(4.0, 0.0, 2.0, 2.0)], rays=[(0.0, 0.0, 1.0, 0.0), (4.0, -5.0, 0.0, 1.0)])
    assert (t, b, f, n) == ([3.0, 4.0], [0, 0], [1, 2], [[-1.0, 0.0], [0.0, -1.0]])
    # an obstacle of the other orientation: the same hit, edge indices of the reversed list
    t, b, f, n = cast(obst=[box(4.0, 0.0, 2.0, 2.0)[::-1]], rays=[(0.0, 0.0, 1.0, 0.0)])
    assert (t, b, f, n) == ([3.0], [0], [1], [[-1.0, 0.0]])


def test_origin_inside_a_body_sees_the_next_body():
    t, b, _, _ = cast(circles=[(0.0, 0.0, 1.0), (5.0, 0.0, 1.0)], rays=[(0.0, 0.0, 1.0, 0.0)])
    assert (t, b) == ([4.0], [1])
    t, b, _, n = cast(circles=[(5.0, 0.0, 1.0)], polys=[box(0.0, 0.0, 2.0, 2.0)], rays=[(0.0, 0.0, 1.0, 0.0)])
    assert (t, b, n) == ([4.0], [0], [[-1.0, 0.0]])
    t, b, _, _ = cast(polys=[box(0.0, 0.0, 2.0, 2.0)], rays=[(0.0, 0.0, 1.0, 0.0)])
    assert (t, b) == ([100.0], [-1])


def test_ray_parallel_to_an_edge():
    # outside the top edge's line: a miss; on its line: the edge is ignored and the ray enters through the left edge
    t, b, f, n = cast(polys=[box(4.0, 0.0, 2.0, 2.0)], rays=[(0.0, 2.0, 1.0, 0.0), (0.0, 1.0, 1.0, 0.0)])
    assert (t, b, f, n) == ([100.0, 3.0], [-1, 0], [-1, 1], [[0.0, 0.0], [-1.0, 0.0]])


def test_ray_through_a_vertex_the_first_edge_wins():
    # (0, 0) -> (1, 1) enters the box [1, 2]^2 at its corner: left (edge 1) and bottom (edge 2) tie, edge 1 wins
    t, b, f, n = cast(polys=[box(1.5, 1.5, 1.0, 1.0)], rays=[(0.0, 0.0, 1.0, 1.0)])
    assert b == [0] and f == [1] and n == [[-1.0, 0.0]]
    assert t[0] == pytest.approx(math.sqrt(2.0), rel=1e-15)


def test_padded_polygon():
    tri = [[3.0, -1.0], [5.0, 0.0], [3.0, 1.0]]
    t3, _, f3, n3 = cast(polys=[tri], rays=[(0.0, 0.0, 1.0, 0.0)])
    t5, _, f5, n5 = cast(polys=[tri + [[3.0, 1.0], [3.0, 1.0]]], rays=[(0.0, 0.0, 1.0, 0.0)])
    assert (t3, f3, n3) == ([3.0], [2], [[-1.0, 0.0]])
    assert (t5, f5, n5) == ([3.0], [4], [[-1.0, 0.0]])             # the repeated vertex's zero-length edges skipped


def test_miss_and_max_dist():
    scene = dict(circles=[(5.0, 0.0, 1.0)])
    assert cast(**scene, rays=[(0.0, 0.0, -1.0, 0.0)])[:3] == ([100.0], [-1], [-1])
    assert cast(**scene, rays=[(0.0, 0.0, 1.0, 0.0)], max_dist=3.5)[:2] == ([3.5], [-1])
    assert cast(**scene, rays=[(0.0, 0.0, 1.0, 0.0)], max_dist=4.0)[:2] == ([4.0], [0])   # t <= max_dist
    assert cast(polys=[box(4.0, 0.0, 2.0, 2.0)], rays=[(0.0, 0.0, 1.0, 0.0)], max_dist=2.5)[:2] == ([2.5], [-1])


def test_zero_direction_and_inactive_bodies():
    c, o = torch.tensor([[[5.0, 0.0]]], dtype=f64), torch.zeros(1, 2, 2, dtype=f64)
    d = torch.tensor([[[0.0, 0.0], [math.nan, 1.0]]], dtype=f64)
    t, b, _, n, _ = ray_ref(c, torch.ones(1, 1, dtype=f64), None, None, o, d, 9.0)
    assert t.tolist() == [[9.0, 9.0]] and b.tolist() == [[-1, -1]] and n.abs().sum() == 0
    t, b, _, _ = cast(circles=[(5.0, 0.0, 1.0), (8.0, 0.0, 1.0)], rays=[(0.0, 0.0, 1.0, 0.0)], active=[False, True])
    assert (t, b) == ([7.0], [1])


def test_equal_distance_the_lower_index_wins():
    t, b, _, _ = cast(circles=[(5.0, 0.5, 1.0), (5.0, -0.5, 1.0)], rays=[(0.0, 0.0, 1.0, 0.0)])
    assert b == [0]
    t, b, _, _ = cast(circles=[(5.0, -0.5, 1.0), (5.0, 0.5, 1.0)], rays=[(0.0, 0.0, 1.0, 0.0)])
    assert b == [0]
    # a circle (body 0) and a box (body 1) both entered at t = 3
    t, b, f, _ = cast(circles=[(4.0, 0.0, 1.0)], polys=[box(4.0, 0.0, 2.0, 2.0)], rays=[(0.0, 0.0, 1.0, 0.0)])
    assert (t, b, f) == ([3.0], [0], [-1])
    t, b, f, _ = cast(polys=[box(4.0, 0.0, 2.0, 2.0)], obst=[box(4.0, 0.0, 2.0, 4.0)], rays=[(0.0, 0.0, 1.0, 0.0)])
    assert (t, b, f) == ([3.0], [0], [1])


def test_mirror_gradients_against_central_differences():
    """d dist / d(origin, direction, circle pos / radius, polygon and obstacle vertices) of the mirror, the choices
    (body, feat) held at the reference's"""
    g = torch.Generator().manual_seed(3)
    c = torch.tensor([[[6.0, 1.0, 1.5], [2.0, 7.0, 1.0]]], dtype=f64)
    pv = torch.tensor([box(-6.0, 1.0, 2.0, 3.0)], dtype=f64).unsqueeze(0)
    ov = torch.tensor([[[1.0, -6.0], [4.0, -5.0], [-2.0, -4.5], [-3.0, -6.5]][::-1]], dtype=f64).unsqueeze(0)
    o = (0.3 * torch.rand(1, 16, 2, generator=g, dtype=f64)).requires_grad_()
    ang = torch.arange(16, dtype=f64) * (2 * math.pi / 16) + 0.05
    d = torch.stack([torch.cos(ang), torch.sin(ang)], 1).unsqueeze(0) * 1.7
    leaves = [o, d.requires_grad_(), c.requires_grad_(), pv.requires_grad_(), ov.requires_grad_()]
    with torch.no_grad():
        u0 = d / d.norm(dim=2, keepdim=True)
        _, body, feat, _, margin = ray_ref(c[..., :2], c[..., 2], pv, ov, o, u0, 50.0)
    assert set(body[0].tolist()) == {-1, 0, 1, 2, 3} and bool((margin > 1e-3).all())   # every body kind hit

    def f(o, d, c, pv, ov):
        u = d / d.norm(dim=2, keepdim=True)
        return BatchedWorldRay(c, pv, ov, o, u, body, feat)

    wt = torch.rand(1, 16, generator=g, dtype=f64)
    y = (f(*leaves) * wt).sum()
    grads = torch.autograd.grad(y, leaves)
    h = 1e-6
    for k, (x, gx) in enumerate(zip(leaves, grads)):
        flat = x.detach().reshape(-1)
        fd = torch.empty_like(flat)
        for i in range(flat.numel()):
            args = [l.detach() for l in leaves]
            xp, xm = flat.clone(), flat.clone()
            xp[i] += h
            xm[i] -= h
            args[k] = xp.reshape(x.shape)
            yp = (f(*args) * wt).sum()
            args[k] = xm.reshape(x.shape)
            ym = (f(*args) * wt).sum()
            fd[i] = (yp - ym) / (2 * h)
        scale = fd.abs().max().clamp_min(1.0)
        assert float((gx.reshape(-1) - fd).abs().max() / scale) < 1e-6


def BatchedWorldRay(c, pv, ov, o, u, body, feat):
    from lcp_physics_b200.world import BatchedWorld
    return BatchedWorld._ray_torch(stand_in(c, pv, ov), o, u, body, feat, 50.0, pv)[0]
