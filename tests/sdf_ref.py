"""Brute-force reference of BatchedWorld's signed distances (lcpb200_signed_distance), independent of the kernel and of
the torch mirror in world.py: dense [B, Q, bodies(, V)] tensors, the rule of include/lcpb200.h evaluated for every
point x body x edge, then the smallest distance with ties to the lower body index. Runs on any device; test support,
not product code."""
import torch


def _unit(d, n2):
    """d / sqrt(n2), 0 where n2 == 0"""
    nz = n2 > 0
    return torch.where(nz.unsqueeze(-1), d / torch.where(nz, n2, torch.ones_like(n2)).sqrt().unsqueeze(-1),
                       torch.zeros_like(d))


def _circles(x, pos, rad):
    """sdf [B,Q,nb] and normals [B,Q,nb,2]; a circle makes no discrete choice"""
    d = x.unsqueeze(2) - pos.unsqueeze(1)                                    # [B,Q,nb,2]
    n2 = (d * d).sum(3)
    return n2.sqrt() - rad.unsqueeze(1), _unit(d, n2)


def _polygons(x, polys):
    """sdf [B,Q,P], feat [B,Q,P] (e outside, 256 + e inside), normals [B,Q,P,2] and the margin of each polygon's own
    choices [B,Q,P]: |max s_e| (inside / outside), and the gap to the runner-up edge (inside: the second largest s_e;
    outside: the second smallest |x - q_e| among edges not tied exactly with the nearest, since the two edges that meet
    at a vertex tie by construction in its region)"""
    nxt = torch.roll(polys, -1, dims=2)
    area = (polys[..., 0] * nxt[..., 1] - polys[..., 1] * nxt[..., 0]).sum(2)
    orient = torch.where(area > 0, 1.0, -1.0).to(polys.dtype).unsqueeze(2)    # [B,P,1]
    E = nxt - polys                                                          # [B,P,V,2]
    ee = (E * E).sum(3)
    ok = ee.sqrt() > 0                                                       # zero-length padding edges are skipped
    ee1 = torch.where(ok, ee, torch.ones_like(ee))
    ln = ee1.sqrt()
    n = torch.stack([orient * E[..., 1] / ln, -orient * E[..., 0] / ln], 3)   # outward unit normals
    okb = ok.unsqueeze(1)
    w = x[:, :, None, None, :] - polys.unsqueeze(1)                          # [B,Q,P,V,2]
    s = torch.where(okb, (n.unsqueeze(1) * w).sum(4), -torch.inf)             # [B,Q,P,V]
    smax = s.max(3).values
    emax = ((s == smax.unsqueeze(3)) & okb).to(torch.int8).argmax(3)          # the first edge of the largest s_e
    inside = smax <= 0
    t = ((w * E.unsqueeze(1)).sum(4) / ee1.unsqueeze(1)).unsqueeze(4)
    P0, P1 = polys.unsqueeze(1), nxt.unsqueeze(1)
    q = torch.where(t <= 0, P0, torch.where(t >= 1, P1, P0 + t * E.unsqueeze(1)))
    dq = x[:, :, None, None, :] - q
    d2 = torch.where(okb, (dq * dq).sum(4), torch.inf)
    dmin = d2.min(3).values
    emin = ((d2 == dmin.unsqueeze(3)) & okb).to(torch.int8).argmax(3)       # the first edge of the smallest distance
    sdf = torch.where(inside, smax, dmin.sqrt())
    feat = torch.where(inside, 256 + emax, emin)
    g = lambda a, i: torch.gather(a, 3, i[..., None, None].expand(*i.shape, 1, 2)).squeeze(3)
    n_in = g(n.unsqueeze(1).expand(-1, x.shape[1], -1, -1, -1), emax)
    dsel = g(dq, emin)
    normal = torch.where(inside.unsqueeze(3), n_in, _unit(dsel, (dsel * dsel).sum(3)))
    s2 = s.topk(2, dim=3).values[..., 1] if s.shape[3] >= 2 else torch.full_like(smax, -torch.inf)
    d_other = torch.where(d2 == dmin.unsqueeze(3), torch.inf, d2).min(3).values
    gap = torch.where(inside, smax - s2, d_other.sqrt() - dmin.sqrt())
    return sdf, feat, normal, torch.minimum(smax.abs(), gap)


def sdf_ref(pos, rad, pverts, overts, points, max_dist, active=None, chunk=256):
    """The signed distances of points [B,Q,2] to circles pos [B,nb,2] / rad [B,nb], dynamic polygons pverts [B,np,V,2]
    and obstacles overts [B,no,V,2] (None: none), active [B,nt] bool or None. Returns (sdf [B,Q], body [B,Q] int64,
    feat [B,Q] int64, normal [B,Q,2], margin [B,Q]): margin is the smallest distance of any discrete decision of the point
    from its threshold (the gap to the second-nearest body, max_dist, and the chosen polygon's inside / outside switch
    and runner-up edge), so that a margin far above round-off certifies that the choice is robust."""
    B, Q, _ = points.shape
    dev = points.device
    nb = pos.shape[1] if pos is not None else 0
    groups = [g for g in (pverts, overts) if g is not None and g.shape[1] > 0]
    polys = torch.cat(groups, 1) if groups else None
    outs = []
    for r0 in range(0, Q, chunk):
        x = points[:, r0:r0 + chunk]
        Qc = x.shape[1]
        valid = torch.isfinite(x).all(2)
        xs = torch.where(valid.unsqueeze(2), x, torch.zeros_like(x))
        ss, ns, fs, ms = [], [], [], []
        if nb:
            s, n = _circles(xs, pos, rad)
            ss.append(s); ns.append(n); fs.append(torch.full_like(s, -1, dtype=torch.int64))
            ms.append(torch.full_like(s, torch.inf))
        if polys is not None:
            s, f, n, m = _polygons(xs, polys)
            ss.append(s); ns.append(n); fs.append(f.long()); ms.append(m)
        S, N, F, M = torch.cat(ss, 2), torch.cat(ns, 2), torch.cat(fs, 2), torch.cat(ms, 2)
        if active is not None:
            S = torch.where(active.to(dev).unsqueeze(1), S, torch.inf)
        S = torch.where(valid.unsqueeze(2), S, torch.inf)
        best = S.min(2).values
        body = (S == best.unsqueeze(2)).to(torch.int8).argmax(2)                # the first (lowest) index of a tie
        hit = best <= max_dist
        second = S.topk(2, dim=2, largest=False).values[..., 1] if S.shape[2] >= 2 else torch.full_like(best, torch.inf)
        own = torch.gather(M, 2, body.unsqueeze(2)).squeeze(2)
        gap = torch.where(torch.isfinite(best), second - best, torch.inf)
        margin = torch.where(valid, torch.minimum(torch.minimum(gap, (best - max_dist).abs()),
                                                  torch.where(hit, own, torch.inf)), torch.inf)
        feat = torch.gather(F, 2, body.unsqueeze(2)).squeeze(2)
        normal = torch.gather(N, 2, body[..., None, None].expand(B, Qc, 1, 2)).squeeze(2)
        outs.append((torch.where(hit, best, torch.full_like(best, max_dist)), torch.where(hit, body, -1),
                     torch.where(hit, feat, -1), torch.where(hit.unsqueeze(2), normal, torch.zeros_like(normal)),
                     margin))
    return tuple(torch.cat(o, 1) for o in zip(*outs))
