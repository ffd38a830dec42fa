"""Brute-force reference of BatchedWorld's shape casts and sweeps (lcpb200_shapecast), independent of the kernel's
face / vertex formulation. Every (query, body) pair is a convex function f(t) along the motion:
  shape casts:  f(t) = sdf_body(o + t u) - r;
  sweeps:       f(t) = sdf_M(t u) - (R_A + R_B) on the Minkowski difference M = conv{b_j - a_i} (scipy ConvexHull, as
                in tests/distance_ref.py), a circle being its centre with its radius.
f is minimised on [0, limit] by golden sections; a miss if the minimum is > 0 (or if f(0) < 0: the bodies overlap at
the start, or f(0) == 0 and the motion does not head into the body); else the first root by bisection on [0, t_min].
The minimum over bodies wins, ties to the lower index. Runs on the CPU in float64; test support, not product code."""
import numpy as np
import torch
from scipy.spatial import ConvexHull

from tests.sdf_ref import _polygons

f64 = torch.float64


class Targets:
    """N convex targets: a point c [N, 2] (is_point) or a polygon P [N, V, 2], inflated by R [N]"""

    def __init__(self, c, P, is_point, R):
        self.c, self.P, self.is_point, self.R = c, P, is_point, R

    def sdf(self, x):
        """(sdf - R, unit sdf gradient) at points x [N, 2]"""
        d = x - self.c
        ln = d.norm(dim=1)
        s = ln
        n = torch.where((ln > 0).unsqueeze(1), d / ln.clamp_min(1e-300).unsqueeze(1), torch.zeros_like(d))
        if self.P is not None:
            ps, _, pn, _ = _polygons(x.unsqueeze(1), self.P.unsqueeze(1))
            s = torch.where(self.is_point, s, ps[:, 0, 0])
            n = torch.where(self.is_point.unsqueeze(1), n, pn[:, 0, 0])
        return s - self.R, n


def first_contact(tg, x0, u, limit, iters=100):
    """t [N] (inf: a miss), the sdf normal at the contact [N, 2] and the margin [N] of the ray x0 + t u, t in
    [0, limit], against the targets"""
    N = x0.shape[0]
    f = lambda t: tg.sdf(x0 + t.unsqueeze(1) * u)[0]
    a, b = torch.zeros(N, dtype=f64), limit.clone()
    g = (np.sqrt(5.0) - 1) / 2
    c_, d_ = b - g * (b - a), a + g * (b - a)
    fc, fd = f(c_), f(d_)
    for _ in range(iters):
        left = fc < fd
        b = torch.where(left, d_, b)
        a = torch.where(left, a, c_)
        c2, d2 = b - g * (b - a), a + g * (b - a)
        nc, nd = torch.where(left, c2, d_), torch.where(left, c_, d2)
        fnc = f(nc)
        fnd = f(nd)
        c_, d_, fc, fd = nc, nd, fnc, fnd
    cand = torch.stack([torch.zeros(N, dtype=f64), c_, d_, limit], 1)
    fv = torch.stack([f(cand[:, k]) for k in range(4)], 1)
    k = fv.argmin(1)
    tmin = cand.gather(1, k.unsqueeze(1)).squeeze(1)
    fmin = fv.gather(1, k.unsqueeze(1)).squeeze(1)
    f0, n0 = tg.sdf(x0)
    slope0 = (n0 * u).sum(1)
    hit = (fmin <= 0) & ((f0 > 0) | ((f0 == 0) & (slope0 < 0)))
    lo, hi = torch.zeros(N, dtype=f64), torch.where(hit, tmin, torch.zeros_like(tmin))
    for _ in range(iters):
        mid = 0.5 * (lo + hi)
        below = f(mid) <= 0
        lo, hi = torch.where(below, lo, mid), torch.where(below, mid, hi)
    t = torch.where(hit, torch.where(f0 == 0, torch.zeros_like(hi), hi), torch.inf)
    th = torch.where(hit, t, 0.0)
    _, n = tg.sdf(x0 + th.unsqueeze(1) * u)
    # a root exactly on a polygon's boundary (no inflation) can read the outside branch at zero distance, whose normal
    # is zero: just inside, the normal is the face's
    _, n_in = tg.sdf(x0 + (th + 1e-9 * th.clamp_min(1.0)).unsqueeze(1) * u)
    n = torch.where((n == 0).all(1, keepdim=True), n_in, n)
    slope = (n * u).sum(1).abs()
    margin = torch.minimum(f0.abs(), torch.where(hit, torch.minimum(slope, (t - limit).abs()), fmin.abs()))
    return t, n, margin


def _best(t, n, margin, limit):
    """the nearest body of t [M, nt] within limit [M] (ties to the lower index): (t, body (-1: none), normal [M, 2] (the
    targets' sdf normal), margin: also the gap to the runner-up and to the limit)"""
    M, nt = t.shape
    best = t.min(1).values
    body = (t == best.unsqueeze(1)).to(torch.int8).argmax(1)
    second = t.topk(2, dim=1, largest=False).values[:, 1] if nt >= 2 else torch.full_like(best, torch.inf)
    own = margin.gather(1, body.unsqueeze(1)).squeeze(1)
    ok = best <= limit
    gap = torch.where(torch.isfinite(best), second - best, torch.inf)
    mg = torch.minimum(torch.minimum(gap, own), (best - limit).abs())
    mg = torch.minimum(mg, margin.min(1).values)               # a grazing miss or an overlap decision anywhere
    normal = n[torch.arange(M), body]
    return (torch.where(ok, best, limit), torch.where(ok, body, -1),
            torch.where(ok.unsqueeze(1), normal, torch.zeros_like(normal)), mg)


def _all_polys(pverts, overts):
    groups = [g.double() for g in (pverts, overts) if g is not None and g.shape[1] > 0]
    return torch.cat(groups, 1) if groups else None


def shapecast_ref(pos, rad, pverts, overts, origin, u, radius, max_dist, active=None):
    """Disk casts: origin / u [B, K, 2] (u of unit length), radius [B, K], against circles pos [B, nb, 2] / rad [B, nb],
    polygons pverts [B, np, V, 2] and obstacles overts [B, no, V, 2] (None: none), active [B, nt] bool or None.
    Returns (dist [B, K], body [B, K], normal [B, K, 2]: the hit body's outward normal, margin [B, K])."""
    B, K, _ = origin.shape
    nb = pos.shape[1] if pos is not None else 0
    polys = _all_polys(pverts, overts)
    nt = nb + (0 if polys is None else polys.shape[1])
    sc = torch.arange(B).repeat_interleave(K * nt)
    j = torch.arange(nt).repeat(B * K)
    o = origin.double().repeat_interleave(nt, 1).reshape(-1, 2)
    uu = u.double().repeat_interleave(nt, 1).reshape(-1, 2)
    r = radius.double().repeat_interleave(nt, 1).reshape(-1)
    is_c = j < nb
    c = torch.zeros(o.shape, dtype=f64)
    R = r.clone()
    if nb:
        ci = torch.where(is_c, j, 0)
        c = pos.double()[sc, ci]
        R = torch.where(is_c, rad.double()[sc, ci] + r, r)
    P = polys[sc, torch.where(is_c, 0, j - nb)] if polys is not None else None
    t, n, m = first_contact(Targets(c, P, is_c, R), o, uu, torch.full_like(r, max_dist))
    if active is not None:
        t = torch.where(active[sc, j], t, torch.inf)
        m = torch.where(active[sc, j], m, torch.inf)
    d, body, normal, margin = _best(t.reshape(B * K, nt), n.reshape(B * K, nt, 2), m.reshape(B * K, nt),
                                    torch.full((B * K,), max_dist, dtype=f64))
    return d.reshape(B, K), body.reshape(B, K), normal.reshape(B, K, 2), margin.reshape(B, K)


def _shape(pos, rad, polys, nb, s, b):
    """points [n, 2] and radius of body b of scene s: a circle's centre, or a polygon's vertices"""
    if b < nb:
        return pos[s, b].double().reshape(1, 2), float(rad[s, b])
    return polys[s, b - nb], 0.0


def sweep_ref(pos, rad, pverts, overts, bodies, disp, active=None, excluded=None):
    """Sweeps of bodies [B, K] (long) by disp [B, K, 2] against every other body (inactive ones and the pairs of
    excluded [B, nt, nt] bool skipped). Returns (frac [B, K], body [B, K], normal [B, K, 2]: from the mover towards
    the hit body, margin [B, K], in units of distance)."""
    B, K = bodies.shape
    nb = pos.shape[1] if pos is not None else 0
    polys = _all_polys(pverts, overts)
    nt = nb + (0 if polys is None else polys.shape[1])
    disp = disp.double()
    L = disp.norm(dim=2)
    u = disp / torch.where(L > 0, L, torch.ones_like(L)).unsqueeze(2)
    rows = []
    for s in range(B):
        for k in range(K):
            a = int(bodies[s, k])
            PA, RA = _shape(pos, rad, polys, nb, s, a)
            for j in range(nt):
                PB, RB = _shape(pos, rad, polys, nb, s, j)
                pts = (PB[None, :, :] - PA[:, None, :]).reshape(-1, 2)
                if pts.shape[0] == 1:
                    rows.append((pts[0], None, RA + RB))
                else:
                    h = ConvexHull(pts.numpy())
                    rows.append((pts[0], pts[torch.from_numpy(h.vertices)], RA + RB))
    V = max([1] + [r[1].shape[0] for r in rows if r[1] is not None])
    N = len(rows)
    c = torch.stack([r[0] for r in rows])
    is_point = torch.tensor([r[1] is None for r in rows])
    P = torch.zeros(N, V, 2, dtype=f64)
    for i, r in enumerate(rows):
        if r[1] is not None:
            P[i, :r[1].shape[0]] = r[1]
            P[i, r[1].shape[0]:] = r[1][-1]
    R = torch.tensor([r[2] for r in rows], dtype=f64)
    uu = u.reshape(-1, 2).repeat_interleave(nt, 0)
    lim = L.reshape(-1).repeat_interleave(nt)
    t, n, m = first_contact(Targets(c, P if V > 1 else None, is_point, R), torch.zeros(N, 2, dtype=f64), uu, lim)
    t, n, m = t.reshape(B, K, nt), -n.reshape(B, K, nt, 2), m.reshape(B, K, nt)
    cand = torch.arange(nt).expand(B, K, nt)
    bad = cand == bodies.unsqueeze(2)
    if active is not None:
        bad = bad | ~active.unsqueeze(1).expand(B, K, nt) | ~torch.gather(active, 1, bodies).unsqueeze(2)
    if excluded is not None:
        bad = bad | torch.gather(excluded, 1, bodies.unsqueeze(2).expand(B, K, nt))
    bad = bad | (L == 0).unsqueeze(2)
    t = torch.where(bad, torch.inf, t)
    m = torch.where(bad, torch.inf, m)
    d, body, normal, margin = _best(t.reshape(B * K, nt), n.reshape(B * K, nt, 2), m.reshape(B * K, nt), L.reshape(-1))
    frac = torch.where(body >= 0, d / torch.where(L.reshape(-1) > 0, L.reshape(-1), 1.0), 1.0)
    return frac.reshape(B, K), body.reshape(B, K), normal.reshape(B, K, 2), margin.reshape(B, K)
