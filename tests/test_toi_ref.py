"""CPU: the time-of-impact rule of lcpb200_time_of_impact on hand-worked cases, for the brute-force reference
(tests/toi_ref.py) and the torch mirror that BatchedWorld.time_of_impact / first_impact differentiate through
(BatchedWorld._impact_torch, called here on a stand-in for the world's state with the kernel's choices worked out by
hand); the mirror's implicit-function gradients against central differences of the reference."""
import math
import types

import pytest
import torch

from tests.sweep_ref import sweep_ref
from tests.test_sdf_ref import box
from tests.toi_ref import toi_ref

f64 = torch.float64


def feat(tf, vtx=0, src_b=0):
    """the packing of lcpb200_body_distance's feat"""
    return tf | vtx << 9 | src_b << 17


def stand_in(circles, polys, rot, obst):
    """the attributes of BatchedWorld that _impact_torch reads: circles [1, nb, 3], polygons [1, np, V, 2] at rotation
    rot [1, np], obstacles [1, no, V, 2] or None"""
    from lcp_physics_b200.world import BatchedWorld, polygon_centroid
    nb, np_ = circles.shape[1], 0 if polys is None else polys.shape[1]
    p = torch.cat([torch.zeros(1, nb, 1, dtype=f64), circles[..., :2]], 2)
    w = types.SimpleNamespace(nb=nb, np=np_, no=0 if obst is None else obst.shape[1], rad=circles[..., 2], ov=obst,
                              dtype=f64, device=torch.device("cpu"))
    w.nv = max([t.shape[2] for t in (polys, obst) if t is not None] + [0])
    if np_:
        cen = polygon_centroid(polys)
        rel = polys - cen.unsqueeze(2)
        c, s = torch.cos(rot).unsqueeze(2), torch.sin(rot).unsqueeze(2)
        w.plocal = torch.stack([c * rel[..., 0] + s * rel[..., 1], -s * rel[..., 0] + c * rel[..., 1]], 3)
        p = torch.cat([p, torch.cat([rot.unsqueeze(2), cen], 2)], 1)
    w.p, w.nd = p, nb + np_
    for name in ("_vertices_at", "_distance_torch", "_sdf_torch", "_impact_torch"):
        setattr(w, name, (lambda f: lambda *a: f(w, *a))(getattr(BatchedWorld, name)))
    return w


def run(circles=(), polys=(), obst=(), motion=(), pairs=(), feats=(), gap=0.0, skip=None):
    """one scene; returns the reference's (frac, body, dist, normal, margin) and the mirror's outputs on the hand
    feats (None for a miss), checked against each other where the margin is wide"""
    c = torch.tensor(circles, dtype=f64).reshape(1, -1, 3)
    pv = torch.tensor(polys, dtype=f64).reshape(1, len(polys), -1, 2) if polys else None
    ov = torch.tensor(obst, dtype=f64).reshape(1, len(obst), -1, 2) if obst else None
    w = stand_in(c, pv, torch.zeros(1, 0 if pv is None else pv.shape[1], dtype=f64), ov)
    m = torch.tensor(motion, dtype=f64).reshape(1, -1, 3)
    pcen = w.p[:, w.nb:, 1:] if w.np else None
    ref = toi_ref(c[..., :2], c[..., 2], pv, pcen, ov, m, [(0, a, b) for a, b in pairs], gap, skip)
    fs = torch.tensor([[-1 if f is None else f for f in feats]])
    assert [b >= 0 for b in ref[1]] == [f is not None for f in feats]
    ba = torch.tensor([[a for a, _ in pairs]])
    bo = torch.tensor([ref[1]])
    out = w._impact_torch(ba, bo, fs, torch.tensor([ref[0]], dtype=f64), m)
    for k in range(len(pairs)):
        if ref[4][k] > 1e-6 and ref[1][k] >= 0:
            assert float(out[2][0, k]) == pytest.approx(ref[2][k], abs=1e-9)
            if ref[2][k] > 1e-6:            # at d = 0 the outside normal of a vertex is the direction of x - q
                assert torch.allclose(out[3][0, k], ref[3][k], atol=1e-7)
    return ref, [t[0] for t in out]


def test_circles_head_on_and_oblique():
    ref, out = run(circles=[(0.0, 0.0, 1.0), (5.0, 0.0, 1.0), (5.0, 1.0, 1.0)],
                   motion=[(0.0, 2.0, 0.0), (0.0, -2.0, 0.0), (0.0, -6.0, 0.0)], pairs=[(0, 1), (1, 2), (0, 2)],
                   feats=[feat(0), None, feat(0)])
    # head on: d = 3 - 4 tau; (1, 2) move apart; oblique: |(5 - 8 tau, 1)| = 2
    assert ref[0][0] == pytest.approx(0.75, abs=1e-12) and ref[1] == [1, -1, 2]
    assert ref[0][2] == pytest.approx((5 - math.sqrt(3)) / 8, abs=1e-12)
    assert out[0].tolist() == ref[0]
    assert out[4][0].tolist() == pytest.approx([2.5, 0.0], abs=1e-12)          # point_a on A, centred at (1.5, 0)
    assert out[5][0].tolist() == pytest.approx([2.5, 0.0], abs=1e-12)
    assert out[3][1].tolist() == [0.0, 0.0] and float(out[0][1]) == 1.0


def test_rod_rotating_in_place_into_a_ball():
    # a rod of half-width 0.05 turning a quarter turn about its centre; its top face reaches the ball of radius 0.3
    # at (0, 1.5) when 1.5 cos(theta) = 0.35
    ref, out = run(circles=[(0.0, 1.5, 0.3)], polys=[box(0.0, 0.0, 4.0, 0.1)],
                   motion=[(0.0, 0.0, 0.0), (math.pi / 2, 0.0, 0.0)], pairs=[(1, 0)], feats=[feat(0, 0, 1)])
    tau = math.acos(0.35 / 1.5) / (math.pi / 2)
    assert ref[0][0] == pytest.approx(tau, abs=1e-12) and ref[1] == [0]
    th = tau * math.pi / 2
    assert out[3][0].tolist() == pytest.approx([-math.sin(th), math.cos(th)], abs=1e-9)


def test_square_corner_rotating_into_a_face():
    # the corner (1, -1) of a 2 x 2 square turning about its centre comes within gap 0.1 of the wall x = 1.2 when
    # sqrt(2) cos(theta - pi / 4) = 1.1
    ref, out = run(polys=[box(0.0, 0.0, 2.0, 2.0)], obst=[box(2.2, 0.0, 2.0, 6.0)], motion=[(0.5, 0.0, 0.0)],
                   pairs=[(0, 1)], feats=[feat(1, 3, 0)], gap=0.1)
    tau = (math.pi / 4 - math.acos(1.1 / math.sqrt(2))) / 0.5
    assert ref[0][0] == pytest.approx(tau, abs=1e-12) and ref[1] == [1]
    assert out[3][0].tolist() == pytest.approx([1.0, 0.0], abs=1e-12)
    assert out[4][0, 0].item() == pytest.approx(1.1, abs=1e-12) and out[2][0].item() == pytest.approx(0.1)


def test_translating_polygons_equal_the_sweep_of_the_relative_displacement():
    a, b = box(0.0, 0.0, 2.0, 2.0), [[6.0, 0.5], [5.0, 1.5], [4.0, 0.5], [5.0, -0.5]]
    ref, _ = run(polys=[a, b], motion=[(0.0, 3.0, 0.2), (0.0, -2.0, 0.0)], pairs=[(0, 1)], feats=[feat(3, 2, 1)])
    pv = torch.tensor([[a, b]], dtype=f64)
    fr, body, _, _ = sweep_ref(torch.zeros(1, 0, 2, dtype=f64), torch.zeros(1, 0, dtype=f64), pv, None,
                               torch.tensor([[0]]), torch.tensor([[[5.0, 0.2]]], dtype=f64))
    assert int(body[0, 0]) == 1 and ref[0][0] == pytest.approx(float(fr[0, 0]), abs=1e-12)


def test_touching_overlapping_and_skipped_pairs():
    circles = [(0.0, 0.0, 1.0), (2.0, 0.0, 1.0), (0.0, 1.5, 1.0), (10.0, 0.0, 1.0)]
    # 0 touches 1: closing reads tau 0, leaving misses; 0 overlaps 2: never seen; still bodies: a miss
    ref, out = run(circles=circles, motion=[(0.0, 1.0, 0.0), (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), (0.0, 0.0, 0.0)],
                   pairs=[(0, 1), (0, 2), (2, 3)], feats=[feat(0), None, None])
    assert ref[0] == [0.0, 1.0, 1.0] and ref[1] == [1, -1, -1]
    assert float(out[0][0]) == 0.0 and out[3][0].tolist() == [1.0, 0.0]
    ref, _ = run(circles=circles, motion=[(0.0, -1.0, 0.0)] + [(0.0, 0.0, 0.0)] * 3, pairs=[(0, 1)], feats=[None])
    assert ref[1] == [-1]
    # skip above the starting distance 6 hides body 3 from body 1; gap 0.5 stops at d = 0.5
    ref, _ = run(circles=circles, motion=[(0.0, 0.0, 0.0), (0.0, 8.0, 0.0)] + [(0.0, 0.0, 0.0)] * 2,
                 pairs=[(1, 3)], feats=[None], gap=0.5, skip=6.5)
    assert ref[1] == [-1]
    ref, _ = run(circles=circles, motion=[(0.0, 0.0, 0.0), (0.0, 8.0, 0.0)] + [(0.0, 0.0, 0.0)] * 2,
                 pairs=[(1, 3)], feats=[feat(0)], gap=0.5)
    assert ref[1] == [3] and ref[0][0] == pytest.approx(5.5 / 8, abs=1e-12) and ref[2][0] == pytest.approx(0.5)


def test_mirror_gradients_against_central_differences():
    """d(frac, dist, normal, witnesses) / d(motion, circles, polygons' vertices, obstacles' vertices) of the mirror at
    the reference's tau, the choices held, against central differences of the reference's tau through the mirror; gap
    0.05 keeps the normals away from d = 0, where a vertex's outside normal has no direction"""
    circles = torch.tensor([[[0.0, 0.0, 1.0], [5.0, 0.5, 1.2], [-10.0, 1.5, 0.3], [9.0, 2.0, 0.5]]], dtype=f64)
    polys = torch.tensor([[box(-10.0, 0.0, 4.0, 0.1), box(10.0, 0.0, 2.0, 2.0)]], dtype=f64)
    obst = torch.tensor([[box(12.2, 0.0, 2.0, 6.0)]], dtype=f64)
    motion = torch.tensor([[[0.0, 2.0, 0.3], [0.0, -2.0, 0.0], [0.0, 0.1, -0.2], [0.0, 3.0, 0.2],
                            [1.5, 0.1, 0.05], [0.5, 0.05, 0.1]]], dtype=f64)
    pairs = [(0, 1), (4, 2), (5, 6), (3, 6)]
    fs = torch.tensor([[feat(0), feat(0, 0, 1), feat(1, 3, 0), feat(1)]])
    ba = torch.tensor([[a for a, _ in pairs]])

    def reference(c_, pv_, ov_, m_):
        w = stand_in(c_, pv_, torch.zeros(1, 2, dtype=f64), ov_)
        r = toi_ref(c_[..., :2], c_[..., 2], pv_, w.p[:, 4:, 1:], ov_, m_, [(0, a, b) for a, b in pairs], gap=0.05)
        return w, r

    w, r = reference(circles, polys, obst, motion)
    assert r[1] == [1, 2, 6, 6] and min(r[4]) > 1e-3 and min(r[0]) > 0.05, r

    def f(c_, pv_, ov_, m_, tau):
        w = stand_in(c_, pv_, torch.zeros(1, 2, dtype=f64), ov_)
        out = w._impact_torch(ba, torch.tensor([r[1]]), fs, tau, m_)
        return torch.cat([out[0].reshape(-1), out[2].reshape(-1), out[3].reshape(-1), out[4].reshape(-1),
                          out[5].reshape(-1)])

    leaves = [t.clone().requires_grad_() for t in (circles, polys, obst, motion)]
    y = f(*leaves, torch.tensor([r[0]], dtype=f64))
    assert torch.allclose(y[:4], torch.tensor(r[0], dtype=f64), atol=0)
    wt = torch.rand(y.shape, generator=torch.Generator().manual_seed(3), dtype=f64)
    grads = torch.autograd.grad((y * wt).sum(), leaves)
    h = 1e-6
    for k, (lf, gx) in enumerate(zip(leaves, grads)):
        flat = lf.detach().reshape(-1)
        fd = torch.empty_like(flat)
        for i in range(flat.numel()):
            ys = []
            for sgn in (1.0, -1.0):
                args = [x.detach() for x in leaves]
                xp = flat.clone()
                xp[i] += sgn * h
                args[k] = xp.reshape(lf.shape)
                tau = torch.tensor([reference(*args)[1][0]], dtype=f64)
                ys.append((f(*args, tau) * wt).sum())
            fd[i] = (ys[0] - ys[1]) / (2 * h)
        assert float((gx.reshape(-1) - fd).abs().max() / fd.abs().max().clamp_min(1.0)) < 1e-5, (k, gx, fd)
        assert float(gx.abs().max()) > 0, k
