"""Brute-force reference of BatchedWorld's body distances (lcpb200_body_distance), independent of the kernel's
formulation: polygon pairs through the Minkowski difference M = conv{b_j - a_i} (scipy.spatial.ConvexHull), whose
signed distance at the origin is the pair's distance outside (the Euclidean distance) and the minimum translation
distance inside, with n_AB = minus M's sdf normal at the origin; circle pairs through tests/sdf_ref.py on the centre,
minus the radius. Runs on the CPU in float64; test support, not product code."""
import numpy as np
import torch
from scipy.spatial import ConvexHull

from tests.sdf_ref import sdf_ref


def minkowski(PA, PB):
    """(sdf, sdf normal [2], margin) of the origin w.r.t. conv{b_j - a_i} of polygons PA [V, 2], PB [V, 2] (numpy):
    margin is the gap of the inside / outside switch and, inside, to the runner-up facet"""
    pts = (PB[None, :, :] - PA[:, None, :]).reshape(-1, 2)
    h = ConvexHull(pts)
    off = h.equations[:, 2]                       # n . x + c <= 0 inside: the origin's value is c
    order = np.argsort(-off, kind="stable")
    S = off[order[0]]
    if S <= 0:
        second = off[order[1]] if len(off) > 1 else -np.inf
        return S, h.equations[order[0], :2].copy(), min(abs(S), S - second)
    best, q = np.inf, None
    for i, j in h.simplices:
        a, b = pts[i], pts[j]
        e = b - a
        t = np.clip(-(a @ e) / (e @ e), 0.0, 1.0)
        c = a + t * e
        if c @ c < best:
            best, q = c @ c, c
    d = np.sqrt(best)
    return d, -q / d, abs(S)


def body_sdf(pos, rad, polys, nb, scene, body, x):
    """signed distance and sdf normal of points x [N, 2] to body `body` [N] of scene `scene` [N] (one body each), with
    sdf_ref's margin; pos [B, nb, 2], rad [B, nb], polys [B, P, V, 2] or None"""
    N = x.shape[0]
    s = torch.zeros(N, dtype=x.dtype)
    n = torch.zeros(N, 2, dtype=x.dtype)
    m = torch.full((N,), torch.inf, dtype=x.dtype)
    c = body < nb
    if bool(c.any()):
        ci = torch.where(c, body, 0)
        r = sdf_ref(pos[scene, ci].unsqueeze(1), rad[scene, ci].unsqueeze(1), None, None, x.unsqueeze(1), np.inf)
        s, n = torch.where(c, r[0][:, 0], s), torch.where(c.unsqueeze(1), r[3][:, 0], n)
    if polys is not None and bool((~c).any()):
        pi = torch.where(c, 0, body - nb)
        r = sdf_ref(torch.zeros(N, 0, 2, dtype=x.dtype), torch.zeros(N, 0, dtype=x.dtype), polys[scene, pi].unsqueeze(1),
                    None, x.unsqueeze(1), np.inf)
        s, n = torch.where(c, s, r[0][:, 0]), torch.where(c.unsqueeze(1), n, r[3][:, 0])
        m = torch.where(c, m, r[4][:, 0])
    return s, n, m


def pair_ref(pos, rad, pverts, overts, pairs, max_dist, active=None):
    """Distances of the pairs [B, K, 2] (long, distinct bodies) of the bodies pos [B, nb, 2] / rad [B, nb], pverts
    [B, np, V, 2], overts [B, no, V, 2] (None: none), active [B, nt] bool or None. Returns (dist [B, K], hit [B, K],
    normal [B, K, 2] from the first body towards the second, margin [B, K]: the distance of the pair's decisions from
    their thresholds -- max_dist, the chosen edge's runner-up, the inside / outside switch); misses read max_dist and
    a zero normal."""
    B, K, _ = pairs.shape
    nb = pos.shape[1] if pos is not None else 0
    if pos is None:
        pos, rad = torch.zeros(B, 0, 2, dtype=torch.float64), torch.zeros(B, 0, dtype=torch.float64)
    groups = [g for g in (pverts, overts) if g is not None and g.shape[1] > 0]
    polys = torch.cat(groups, 1).double() if groups else None
    pos, rad = pos.double(), rad.double()
    a, b = pairs[..., 0].reshape(-1), pairs[..., 1].reshape(-1)
    sc = torch.arange(B).repeat_interleave(K)
    N = B * K
    dist = torch.full((N,), np.inf, dtype=torch.float64)
    normal = torch.zeros(N, 2, dtype=torch.float64)
    margin = torch.full((N,), np.inf, dtype=torch.float64)
    ca, cb = a < nb, b < nb
    # a circle's centre is the source, the first body's when both are circles
    src_b = ~ca & cb
    circ = ca | cb
    if bool(circ.any()):
        src, tgt = torch.where(src_b, b, a)[circ], torch.where(src_b, a, b)[circ]
        s_ = sc[circ]
        x = pos[s_, src]
        s, m, mg = body_sdf(pos, rad, polys, nb, s_, tgt, x)
        dist[circ] = s - rad[s_, src]
        normal[circ] = torch.where(src_b[circ].unsqueeze(1), m, -m)
        margin[circ] = mg
    for i in torch.nonzero(~circ).flatten().tolist():
        d, m, mg = minkowski(polys[sc[i], a[i] - nb].numpy(), polys[sc[i], b[i] - nb].numpy())
        dist[i], margin[i] = d, mg
        normal[i] = -torch.from_numpy(m)
    if active is not None:
        on = active[sc, a] & active[sc, b]
        dist = torch.where(on, dist, torch.inf)
    hit = dist <= max_dist
    margin = torch.minimum(margin, (dist - max_dist).abs())
    dist = torch.where(hit, dist, torch.full_like(dist, max_dist))
    normal = torch.where(hit.unsqueeze(1), normal, torch.zeros_like(normal))
    return dist.reshape(B, K), hit.reshape(B, K), normal.reshape(B, K, 2), margin.reshape(B, K)


def nearest_ref(pos, rad, pverts, overts, bodies, max_dist, active=None, excluded=None):
    """The nearest other body of each query body [B, K] (long) over every candidate, inactive ones and the pairs of
    excluded [B, nt, nt] (bool, or None) skipped, ties to the lower index. Returns (dist, body [B, K] (-1: none within
    max_dist), normal, margin: also the gap to the runner-up candidate)."""
    B, K = bodies.shape
    nt = sum(g.shape[1] for g in (pos, pverts, overts) if g is not None)
    cand = torch.arange(nt).expand(B, K, nt)
    q = bodies.unsqueeze(2).expand(B, K, nt)
    pairs = torch.stack([q, torch.where(cand == q, (q + 1) % nt, cand)], 3).reshape(B, K * nt, 2)
    d, hit, n, m = pair_ref(pos, rad, pverts, overts, pairs, np.inf, active)
    d, hit, n, m = d.reshape(B, K, nt), hit.reshape(B, K, nt), n.reshape(B, K, nt, 2), m.reshape(B, K, nt)
    bad = cand == q
    if excluded is not None:
        bad = bad | torch.gather(excluded, 1, bodies.unsqueeze(2).expand(B, K, nt))
    d = torch.where(bad | ~hit, torch.inf, d)
    best = d.min(2).values
    body = (d == best.unsqueeze(2)).to(torch.int8).argmax(2)
    second = d.topk(2, dim=2, largest=False).values[..., 1] if nt >= 2 else torch.full_like(best, torch.inf)
    own = torch.gather(m, 2, body.unsqueeze(2)).squeeze(2)
    ok = best <= max_dist
    margin = torch.minimum(torch.minimum(second - best, own), (best - max_dist).abs())
    normal = torch.gather(n, 2, body[..., None, None].expand(B, K, 1, 2)).squeeze(2)
    return (torch.where(ok, best, torch.full_like(best, max_dist)), torch.where(ok, body, -1),
            torch.where(ok.unsqueeze(2), normal, torch.zeros_like(normal)), margin)
