"""CPU: the body-distance rule of lcpb200_body_distance on hand-worked cases, for the brute-force reference
(tests/distance_ref.py) and the torch mirror that BatchedWorld.distance / nearest differentiate through
(BatchedWorld._distance_torch, called here on a stand-in for the world's state with the kernel's choices worked out by
hand); the mirror's gradients against central differences."""
import math
import types

import pytest
import torch

from tests.distance_ref import nearest_ref, pair_ref
from tests.test_sdf_ref import box

f64 = torch.float64
R2 = math.sqrt(0.5)


def feat(tf, vtx=0, src_b=0):
    """the packing of lcpb200_body_distance's feat"""
    return tf | vtx << 9 | src_b << 17


def stand_in(c, pv, ov):
    """the attributes of BatchedWorld that _distance_torch and _sdf_torch read"""
    from lcp_physics_b200.world import BatchedWorld
    nb = c.shape[1]
    np_ = 0 if pv is None else pv.shape[1]
    p = torch.cat([torch.zeros(1, nb, 1, dtype=f64), c[..., :2]], 2)
    if np_:
        p = torch.cat([p, torch.zeros(1, np_, 3, dtype=f64)], 1)
    nv = max(0 if pv is None else pv.shape[2], 0 if ov is None else ov.shape[2])
    w = types.SimpleNamespace(nb=nb, np=np_, no=0 if ov is None else ov.shape[1], nv=nv, p=p, rad=c[..., 2], ov=ov,
                              dtype=f64, device=torch.device("cpu"))
    w._sdf_torch = lambda *a: BatchedWorld._sdf_torch(w, *a)
    return w


def scene(circles=(), polys=(), obst=()):
    c = torch.tensor(circles, dtype=f64).reshape(1, -1, 3)
    pv = torch.tensor(polys, dtype=f64).reshape(1, len(polys), -1, 2) if polys else None
    ov = torch.tensor(obst, dtype=f64).reshape(1, len(obst), -1, 2) if obst else None
    return c, pv, ov


def choices(c, pv, ov, pairs):
    """the kernel's choices (feat) for pairs [(a, b)] of one scene, by brute force over the rule of lcp_distance.cuh:
    the source point's sdf choices from tests/sdf_ref.py, the separating axis by a loop over faces and vertices"""
    from tests.sdf_ref import sdf_ref
    nb = c.shape[1]
    polys = torch.cat([t for t in (pv, ov) if t is not None], 1)[0] if (pv is not None or ov is not None) else None
    empty = (torch.zeros(1, 0, 2, dtype=f64), torch.zeros(1, 0, dtype=f64))

    def sdf(x, t):
        if t < nb:
            return float((x - c[0, t, :2]).norm() - c[0, t, 2]), 0
        r = sdf_ref(*empty, polys[t - nb][None, None], None, x.reshape(1, 1, 2), 1e300)
        return float(r[0]), int(r[2])

    def sat(P, Q):
        """(S, face, support vertex of Q) over the faces of P: the first face of the largest value, the last vertex"""
        V = P.shape[0]
        o = 1.0 if float((P[:, 0] * P.roll(-1, 0)[:, 1] - P[:, 1] * P.roll(-1, 0)[:, 0]).sum()) > 0 else -1.0
        best = (-math.inf, 0, 0)
        for e in range(V):
            E = P[(e + 1) % V] - P[e]
            if float(E.norm()) == 0:
                continue
            n = torch.stack([o * E[1], -o * E[0]]) / E.norm()
            proj = -(Q @ n)
            sup = max(i for i in range(Q.shape[0]) if proj[i] == proj.max())
            s = float(n @ (Q[sup] - P[e]))
            if s > best[0]:
                best = (s, e, sup)
        return best

    out = []
    for a, b in pairs:
        if a < nb or b < nb:
            src_b = int(a >= nb)
            s, t = (b, a) if src_b else (a, b)
            out.append(feat(sdf(c[0, s, :2], t)[1], 0, src_b))
            continue
        PA, PB = polys[a - nb], polys[b - nb]
        sa, sb = sat(PA, PB), sat(PB, PA)
        if max(sa[0], sb[0]) <= 0:
            out.append(feat(256 + sb[1], sb[2], 0) if sb[0] > sa[0] else feat(256 + sa[1], sa[2], 1))
            continue
        best = None
        for src_b, (S, T) in enumerate(((a, b), (b, a))):
            for i in range(polys.shape[1]):
                d, f = sdf(polys[S - nb, i], T)
                if best is None or d < best[0]:
                    best = (d, feat(f, i, src_b))
        out.append(best[1])
    return out


def check(sc, pairs, max_dist=100.0, active=None):
    """the reference on pairs [(a, b)], and the mirror on the rule's choices; returns the reference's (dist, hit,
    normal) as lists and the mirror's (dist, normal, point_a, point_b); normals are compared where the reference's
    choice is unique (margin > 0)"""
    from lcp_physics_b200.world import BatchedWorld
    c, pv, ov = sc
    pr = torch.tensor(pairs).reshape(1, -1, 2)
    act = None if active is None else torch.tensor(active).reshape(1, -1)
    d, hit, n, margin = pair_ref(c[..., :2], c[..., 2], pv, ov, pr, max_dist, act)
    bo = torch.where(hit, pr[..., 1], -1)
    fs = torch.where(hit, torch.tensor([choices(c, pv, ov, pairs)]), -1)
    m = BatchedWorld._distance_torch(stand_in(c, pv, ov), pr[..., 0], bo, fs, max_dist, pv)
    assert torch.allclose(m[0], d, rtol=1e-15, atol=1e-15), (m[0], d)
    u = (margin > 0).unsqueeze(2)
    assert torch.allclose(m[1] * u, n * u, rtol=1e-15, atol=1e-15), (m[1], n)
    nz = m[1].norm(dim=2) > 0                                            # a zero normal: coincident witnesses
    assert torch.allclose((m[3] - m[2]).norm(dim=2), d.abs() * nz, rtol=1e-15, atol=1e-15)
    return d[0].tolist(), hit[0].tolist(), n[0].tolist(), [t[0].tolist() for t in m]


def close(a, b):
    return a == pytest.approx(b, rel=1e-15, abs=1e-15)


def test_squares_face_to_face_and_corner_to_corner():
    sc = scene(polys=[box(0.0, 0.0, 2.0, 2.0), box(3.0, 0.0, 2.0, 2.0), box(3.0, 3.0, 2.0, 2.0)])
    # A's vertex 0 (1, 1) is 1 from B's vertex (2, 1), where B's edges 0 and 1 meet: edge 0 wins
    d, hit, n, (_, _, pa, pb) = check(sc, [(0, 1), (1, 0), (0, 2)])
    assert d[0] == 1.0 and n[0] == [1.0, 0.0] and pa[0] == [1.0, 1.0] and pb[0] == [2.0, 1.0]
    assert d[1] == 1.0 and n[1] == [-1.0, 0.0] and pa[1] == [2.0, 1.0]
    assert close(d[2], math.sqrt(2.0)) and close(n[2], [R2, R2]) and pa[2] == [1.0, 1.0] and pb[2] == [2.0, 2.0]


def test_rotated_square_dips_into_a_face():
    diamond = [[0.0, 1.25], [-1.0, 2.25], [0.0, 3.25], [1.0, 2.25]]            # vertex 0 is 0.25 below y = 1.5
    sc = scene(polys=[box(0.0, 0.0, 4.0, 3.0), diamond])
    # S from A's top face (edge 0, y = 1.5): B's support vertex 0 at -0.25; B is the source
    d, _, n, (_, _, pa, pb) = check(sc, [(0, 1)])
    assert d == [-0.25] and n == [[0.0, 1.0]]
    assert pa[0] == [0.0, 1.5] and pb[0] == [0.0, 1.25]          # the face's supporting line and the vertex


def test_identical_and_nested_squares():
    sq = box(0.0, 0.0, 2.0, 2.0)
    sc = scene(polys=[sq, sq, box(0.0, 0.0, 1.0, 1.0)])
    # identical: every face gives -2; A's first face wins, B's support vertex the last minimal one (vertex 3 on y = -1)
    d, _, _, (_, mn, pa, pb) = check(sc, [(0, 1)])
    assert choices(*sc, [(0, 1)]) == [feat(256 + 0, 3, 1)]
    assert d == [-2.0] and mn[0] == [0.0, 1.0] and pa[0] == [1.0, 1.0] and pb[0] == [1.0, -1.0]
    # nested: every face ties at -1.5; the first polygon's top face wins, the other's last lowest vertex is the source
    d, _, _, (_, mn, _, _) = check(sc, [(0, 2), (2, 0)])
    assert choices(*sc, [(0, 2), (2, 0)]) == [feat(256 + 0, 3, 1), feat(256 + 0, 3, 1)]
    assert d == [-1.5, -1.5] and mn == [[0.0, 1.0], [0.0, 1.0]]


def test_circle_pairs():
    sc = scene(circles=[(0.0, 0.0, 1.0), (3.0, 4.0, 2.0), (1.0, 0.0, 1.0), (0.0, 0.0, 0.5)])
    d, _, n, (_, _, pa, pb) = check(sc, [(0, 1), (0, 2), (0, 3)])
    assert d == [2.0, -1.0, -1.5]
    assert close(n[0], [0.6, 0.8]) and close(pa[0], [0.6, 0.8]) and close(pb[0], [1.8, 2.4])
    assert n[1] == [1.0, 0.0] and pa[1] == [1.0, 0.0] and pb[1] == [0.0, 0.0]
    assert n[2] == [0.0, 0.0] and pa[2] == [0.0, 0.0] == pb[2]     # coincident centres: a zero normal


def test_circle_and_square():
    sc = scene(circles=[(4.0, 0.0, 1.0), (3.0, 3.0, 1.0), (0.5, 0.0, 0.25)], polys=[box(0.0, 0.0, 2.0, 2.0)])
    d, _, n, (_, _, pa, pb) = check(sc, [(0, 3), (3, 0), (1, 3), (2, 3)])
    assert choices(*sc, [(0, 3), (3, 0), (1, 3), (2, 3)]) == [feat(3), feat(3, 0, 1), feat(0), feat(256 + 3)]
    assert d[:2] == [2.0, 2.0] and n[0] == [-1.0, 0.0] and n[1] == [1.0, 0.0]
    assert pa[0] == [3.0, 0.0] and pb[0] == [1.0, 0.0] and pa[1] == [1.0, 0.0] and pb[1] == [3.0, 0.0]
    assert close(d[2], math.sqrt(8.0) - 1.0) and close(n[2], [-R2, -R2])
    assert d[3] == -0.75 and n[3] == [-1.0, 0.0] and pb[3] == [1.0, 0.0]          # from inside: the right face


def test_padded_polygons_and_reversed_obstacles():
    tri = [[3.0, -1.0], [5.0, 0.0], [3.0, 1.0]]
    padded = tri + [[3.0, 1.0], [3.0, 1.0]]
    sq = box(0.0, 0.0, 2.0, 2.0)
    a = check(scene(polys=[sq + [sq[-1]], padded]), [(0, 1), (1, 0)])
    b = check(scene(polys=[sq], obst=[tri + [tri[-1]]]), [(0, 1), (1, 0)])
    assert a[0] == b[0] == [2.0, 2.0] and a[2] == b[2] == [[1.0, 0.0], [-1.0, 0.0]]
    c = check(scene(polys=[sq], obst=[box(4.0, 0.0, 2.0, 2.0)[::-1]]), [(0, 1)])
    assert c[0] == [2.0] and c[2] == [[1.0, 0.0]]
    # the diamond of test_rotated_square_dips_into_a_face, reversed: the same distance from the same face
    diamond = [[0.0, 1.25], [-1.0, 2.25], [0.0, 3.25], [1.0, 2.25]]
    r = check(scene(polys=[box(0.0, 0.0, 4.0, 3.0)], obst=[diamond[::-1]]), [(0, 1)])
    assert r[0] == [-0.25] and r[2] == [[0.0, 1.0]]


def test_max_dist_boundary_and_inactive_bodies():
    sc = scene(circles=[(0.0, 0.0, 1.0), (5.0, 0.0, 1.0), (2.5, 0.0, 0.5)])
    assert check(sc, [(0, 1)], max_dist=3.0)[:2] == ([3.0], [True])         # d <= max_dist hits
    d, hit, n, (md, mn, pa, pb) = check(sc, [(0, 1)], max_dist=2.5)
    assert (d, hit, n) == ([2.5], [False], [[0.0, 0.0]]) and pa == [[0.0, 0.0]] == pb
    d, hit, _, _ = check(sc, [(0, 2), (0, 1)], active=[True, True, False])
    assert hit == [False, True] and d == [100.0, 3.0]
    nd, nbody, _, _ = nearest_ref(sc[0][..., :2], sc[0][..., 2], None, None, torch.tensor([[0, 1, 2]]), 100.0,
                                  active=torch.tensor([[True, True, False]]))
    assert nbody[0].tolist() == [1, 0, -1] and nd[0].tolist() == [3.0, 3.0, 100.0]


def test_mirror_gradients_against_central_differences():
    """d(dist, normal, point_a, point_b) / d(circles, polygon and obstacle vertices) of the mirror, the choices held"""
    from lcp_physics_b200.world import BatchedWorld
    c = torch.tensor([[[6.0, 1.0, 1.5], [2.0, 7.0, 1.0]]], dtype=f64)
    pv = torch.tensor([[[-5.0, 2.0], [-7.0, 2.5], [-7.5, -0.5], [-5.5, -1.0]]], dtype=f64).unsqueeze(0)
    ov = torch.tensor([[[1.0, -6.0], [4.0, -5.0], [-2.0, -4.5], [-3.0, -6.5]][::-1]], dtype=f64).unsqueeze(0)
    pairs = torch.tensor([[[0, 1], [0, 2], [2, 0], [3, 2], [1, 3], [2, 3]]])
    w = stand_in(c, pv, ov)
    d, hit, n, margin = pair_ref(c[..., :2], c[..., 2], pv, ov, pairs, 100.0)
    assert bool(hit.all()) and bool((margin > 1e-3).all())
    fs = torch.tensor([choices(c, pv, ov, pairs[0].tolist())])
    leaves = [c.clone().requires_grad_(), pv.clone().requires_grad_(), ov.clone().requires_grad_()]

    def f(c_, pv_, ov_):
        w.p = torch.cat([torch.cat([torch.zeros(1, 2, 1, dtype=f64), c_[..., :2]], 2), torch.zeros(1, 1, 3, dtype=f64)],
                        1)
        w.rad, w.ov = c_[..., 2], ov_
        out = BatchedWorld._distance_torch(w, pairs[..., 0], pairs[..., 1], fs, 100.0, pv_)
        return torch.cat([out[0].unsqueeze(2), out[1], out[2], out[3]], 2)

    y = f(*leaves)
    assert torch.allclose(y[..., 0], d, rtol=1e-14, atol=1e-14) and torch.allclose(y[..., 1:3], n, atol=1e-14)
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
