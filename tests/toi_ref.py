"""Brute-force reference of BatchedWorld's times of impact (lcpb200_time_of_impact), independent of conservative
advancement: the pair's distance d(tau) (tests/distance_ref.py) at the bodies' poses at tau, sampled on a dense grid
of [0, 1]; the first sign change of d - gap is then bisected. A pair closer than skip at tau = 0 is not seen, one exactly
at skip only when d falls. Runs on the CPU in float64; test support, not product code."""
import math

import numpy as np
import torch

from tests.distance_ref import pair_ref

f64 = torch.float64


def poses(pos, pverts, pcen, motion, tau):
    """the circles' centres [B, nb, 2] and the polygons' vertices [B, np, V, 2] at tau (a float): c + tau dc + R(tau
    dth)(v - c); motion [B, nb + np, 3] (dth, dx, dy)"""
    nb = pos.shape[1]
    c = pos + tau * motion[:, :nb, 1:]
    if pverts is None:
        return c, None
    m = motion[:, nb:]
    th = tau * m[..., 0:1]
    w = pverts - pcen.unsqueeze(2)
    cs, sn = torch.cos(th), torch.sin(th)
    rot = torch.stack([cs * w[..., 0] - sn * w[..., 1], sn * w[..., 0] + cs * w[..., 1]], 3)
    return c, pcen.unsqueeze(2) + tau * m[:, :, None, 1:] + rot


def pair_toi(pos, rad, pverts, pcen, overts, motion, s, a, b, gap, skip, grid=200, iters=60):
    """(tau, d at tau, normal [2], margin) of the pair (a, b) of scene s; tau = inf on a miss. margin: the smallest of
    |d'| at the root, 1 - tau and d(0) - skip (how far the decision is from switching)"""
    def d(t):
        c, pv = poses(pos[s:s + 1], None if pverts is None else pverts[s:s + 1],
                      None if pcen is None else pcen[s:s + 1], motion[s:s + 1], t)
        dist, _, n, _ = pair_ref(c, rad[s:s + 1], pv, None if overts is None else overts[s:s + 1],
                                 torch.tensor([[[a, b]]]), math.inf)
        return float(dist[0, 0]), n[0, 0]
    still = lambda k: k >= motion.shape[1] or bool((motion[s, k] if k >= pos.shape[1] else motion[s, k, 1:]).eq(0).all())
    if still(a) and still(b):
        return math.inf, 0.0, torch.zeros(2, dtype=f64), math.inf
    d0 = d(0.0)[0]
    h = 1e-7
    slope0 = (d(h)[0] - d0) / h
    if d0 < skip or (d0 == skip and not slope0 < 0):
        return math.inf, 0.0, torch.zeros(2, dtype=f64), abs(d0 - skip)
    if d0 <= gap:
        return 0.0, d0, d(0.0)[1], min(abs(d0 - skip), abs(d0 - gap)) if d0 != skip else abs(slope0)
    ts = np.linspace(0.0, 1.0, grid + 1)
    prev = 0.0
    for t in ts[1:]:
        if d(float(t))[0] <= gap:
            lo, hi = prev, float(t)
            for _ in range(iters):
                mid = 0.5 * (lo + hi)
                if d(mid)[0] <= gap:
                    hi = mid
                else:
                    lo = mid
            dd, n = d(hi)
            slope = (d(hi)[0] - d(max(hi - 1e-6, 0.0))[0]) / min(1e-6, hi) if hi > 0 else slope0
            return hi, dd, n, min(abs(slope), 1.0 - hi, abs(d0 - skip))
        prev = float(t)
    return math.inf, 0.0, torch.zeros(2, dtype=f64), abs(d(1.0)[0] - gap)


def toi_ref(pos, rad, pverts, pcen, overts, motion, queries, gap=0.0, skip=None, first=False, active=None,
            excluded=None):
    """queries: [(scene, a, b)] (pair mode) or [(scene, a)] (first mode: every other body, inactive ones and the pairs
    of excluded [B, nt, nt] skipped, ties to the lower index). Returns lists (frac, body, dist, normal, margin); the
    margin of a first-mode query also holds the gap to the runner-up's tau."""
    skip = gap if skip is None else skip
    nt = pos.shape[1] + sum(0 if g is None else g.shape[1] for g in (pverts, overts))
    on = (lambda s, k: True) if active is None else (lambda s, k: bool(active[s, k]))
    out = []
    for q in queries:
        s, a = q[0], q[1]
        cands = [q[2]] if not first else [j for j in range(nt) if j != a and
                                          (excluded is None or not bool(excluded[s, a, j]))]
        res = []
        for j in cands:
            if not (on(s, a) and on(s, j)):
                continue
            t, dd, n, m = pair_toi(pos, rad, pverts, pcen, overts, motion, s, a, j, gap, skip)
            res.append((t, j, dd, n, m))
        hits = sorted([r for r in res if r[0] <= 1.0], key=lambda r: (r[0], r[1]))
        if not hits:
            mg = min([r[4] for r in res] + [math.inf])
            out.append((1.0, -1, 0.0, torch.zeros(2, dtype=f64), mg))
            continue
        t, j, dd, n, m = hits[0]
        runner = hits[1][0] - t if len(hits) > 1 else math.inf
        out.append((t, j, dd, n, min([m, runner] + [r[4] for r in res if r[0] > 1.0])))
    return [list(x) for x in zip(*out)]
