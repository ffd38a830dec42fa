"""Brute-force reference of BatchedWorld's ray casts (lcpb200_raycast), independent of the kernel and of the torch mirror
in world.py: dense [B, R, bodies(, V)] tensors, the rule of include/lcpb200.h evaluated for every ray x body x edge,
then the nearest hit with ties to the lower body index. Runs on any device; test support, not product code."""
import torch


def _circles(o, u, pos, rad, max_dist):
    """t [B,R,nb] (inf: no hit), normals [B,R,nb,2] and a decision margin [B,R,nb]"""
    w = o.unsqueeze(2) - pos.unsqueeze(1)                                    # [B,R,nb,2]
    b = (u.unsqueeze(2) * w).sum(3)
    r = rad.unsqueeze(1)
    k = (w * w).sum(3) - r * r
    disc = b * b - k
    hit = (k >= 0) & (b < 0) & (disc >= 0)
    t = k / (-b + disc.clamp_min(0).sqrt())
    hit = hit & (t <= max_dist)
    n = (w + t.unsqueeze(3) * u.unsqueeze(2)) / r.unsqueeze(3)
    # the choices flip only where k, disc or t - max_dist change sign (b < 0 vs b >= 0 flips only with disc >= 0, i.e.
    # |k| <= b^2 -- covered by |k| and |disc| together)
    margin = torch.minimum(torch.minimum(k.abs(), disc.abs()), torch.where(hit, (t - max_dist).abs(), torch.inf))
    return torch.where(hit, t, torch.inf), n, margin


def _polygons(o, u, polys, max_dist):
    """t [B,R,P] (inf: no hit), entering edge [B,R,P], its normal [B,R,P,2] and a decision margin [B,R,P]"""
    V = polys.shape[2]
    nxt = torch.roll(polys, -1, dims=2)
    area = (polys[..., 0] * nxt[..., 1] - polys[..., 1] * nxt[..., 0]).sum(2)
    orient = torch.where(area > 0, 1.0, -1.0).to(polys.dtype).unsqueeze(2)    # [B,P,1]
    E = nxt - polys
    ln = E.norm(dim=3)
    ok = ln > 0                                                              # zero-length padding edges are skipped
    l1 = torch.where(ok, ln, torch.ones_like(ln))
    n = torch.stack([orient * E[..., 1] / l1, -orient * E[..., 0] / l1], 3)   # [B,P,V,2] outward unit normals
    rel = polys.unsqueeze(1) - o[:, :, None, None, :]                         # [B,R,P,V,2]
    num = (n.unsqueeze(1) * rel).sum(4)                                      # [B,R,P,V]
    den = (n.unsqueeze(1) * u[:, :, None, None, :]).sum(4)
    okb = ok.unsqueeze(1)
    par_miss = (okb & (den == 0) & (num < 0)).any(3)
    t = num / torch.where(den == 0, torch.ones_like(den), den)
    ent = okb & (den < 0)
    lea = okb & (den > 0)
    te_all = torch.where(ent, t, -torch.inf)
    te = te_all.max(3).values
    fe = ((te_all == te.unsqueeze(3)) & ent).to(torch.int8).argmax(3)         # the first edge of the largest t
    tl = torch.where(lea, t, torch.inf).min(3).values
    has = ent.any(3)
    hit = ~par_miss & has & (te >= 0) & (te <= tl) & (te <= max_dist)
    nsel = torch.gather(n.unsqueeze(1).expand(-1, o.shape[1], -1, -1, -1), 3,
                        fe[..., None, None].expand(*fe.shape, 1, 2)).squeeze(3)
    den_fe = torch.gather(den, 3, fe.unsqueeze(3)).squeeze(3).abs()             # a grazing entry is ill-conditioned
    top2 = te_all.topk(2, dim=3).values if V >= 2 else te_all
    gap = (top2[..., 0] - top2[..., 1]) if V >= 2 else torch.full_like(te, torch.inf)
    margin = torch.where(has & ~par_miss, torch.minimum((te - tl).abs(), te.abs()), torch.inf)
    margin = torch.minimum(margin, torch.where(hit, torch.minimum(torch.minimum(gap, den_fe), (te - max_dist).abs()),
                                                   torch.inf))
    return torch.where(hit, te, torch.inf), fe, nsel, margin


def ray_ref(pos, rad, pverts, overts, origin, direction, max_dist, active=None, chunk=256):
    """The readings of rays origin / direction [B,R,2] (direction of unit length) against circles pos [B,nb,2] /
    rad [B,nb], dynamic polygons pverts [B,np,V,2] and obstacles overts [B,no,V,2] (None: none), active [B,nt] bool or
    None. Returns (t [B,R], body [B,R] int64, feat [B,R] int64, normal [B,R,2], margin [B,R]): margin is the smallest
    distance of any discrete decision of the ray from its threshold (second-nearest hit, discriminants, Cyrus-Beck
    entry / exit, top-two entering edges, incidence of the entering edge), so that a margin far above round-off certifies that the choice is robust."""
    B, R, _ = origin.shape
    dev = origin.device
    nb = pos.shape[1] if pos is not None else 0
    groups = [g for g in (pverts, overts) if g is not None and g.shape[1] > 0]
    polys = torch.cat(groups, 1) if groups else None
    outs = []
    for r0 in range(0, R, chunk):
        o, u = origin[:, r0:r0 + chunk], direction[:, r0:r0 + chunk]
        Rc = o.shape[1]
        valid = torch.isfinite(o).all(2) & torch.isfinite(u).all(2) & ((u * u).sum(2) > 0)
        ts, ns, fs, ms = [], [], [], []
        if nb:
            t, n, m = _circles(o, u, pos, rad, max_dist)
            ts.append(t); ns.append(n); fs.append(torch.full_like(t, -1, dtype=torch.int64)); ms.append(m)
        if polys is not None:
            t, f, n, m = _polygons(o, u, polys, max_dist)
            ts.append(t); ns.append(n); fs.append(f.long()); ms.append(m)
        T, N, F, M = torch.cat(ts, 2), torch.cat(ns, 2), torch.cat(fs, 2), torch.cat(ms, 2)
        if active is not None:
            on = active.to(dev).unsqueeze(1)
            T = torch.where(on, T, torch.inf)
            M = torch.where(on, M, torch.inf)
        T = torch.where(valid.unsqueeze(2), T, torch.inf)
        best = T.min(2).values
        body = (T == best.unsqueeze(2)).to(torch.int8).argmax(2)                # the first (lowest) index of a tie
        hit = torch.isfinite(best)
        second = T.topk(2, dim=2, largest=False).values[..., 1] if T.shape[2] >= 2 else torch.full_like(best, torch.inf)
        margin = torch.minimum(torch.where(valid, M.min(2).values, torch.inf),
                               torch.where(hit, second - best, torch.inf))
        feat = torch.gather(F, 2, body.unsqueeze(2)).squeeze(2)
        normal = torch.gather(N, 2, body[..., None, None].expand(B, Rc, 1, 2)).squeeze(2)
        outs.append((torch.where(hit, best, torch.full_like(best, max_dist)), torch.where(hit, body, -1),
                     torch.where(hit, feat, -1), torch.where(hit.unsqueeze(2), normal, torch.zeros_like(normal)),
                     margin))
    return tuple(torch.cat(x, 1) for x in zip(*outs))
