"""Distances between `BatchedWorld` bodies (lcpb200_body_distance, `distance`, `nearest`), timed on the GPU.

* (a) 1024 piles of 24 balls in a bin of 3 obstacles, `nearest` for all 24 balls:
    kernel      nothing differentiated;
    graph_bwd   the state requiring grad, then a backward pass of the distances' sum;
    brute       a torch brute force (every ball pair, sdf_ref of every centre to the obstacles);
* (b) 256 scenes of 16 hulls (8 vertices) on a floor: `nearest` for all hulls and `distance` over all 120 hull pairs,
  kernel and graph_bwd;
* (c) 256 scenes of two 256-gons (the O(V^2) polygon pair, one thread per pair): `distance` of the pair;
* (d) one 512-ball pile, `nearest` for all balls: kernel, graph_bwd and brute;
* (e) one `nearest` call of (a) against one `step()` of the same worlds.
Legs of a pairing alternate inside every round; prints one JSON line per pairing with the median and the spread
(min, max) of every leg, and the card and its power limit read in the same run.

    python scripts/distance_bench.py [--rounds 5] [--calls 20] [--warmup 3] [--batch 1024]
"""
import argparse
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lcp_physics_b200.scenes import make_ball_pile  # noqa: E402
from lcp_physics_b200.world import BatchedWorld, rect_vertices  # noqa: E402
from scripts.hetero_bench import G, balls, bin_obstacles  # noqa: E402
from scripts.raycast_bench import pairing  # noqa: E402
from tests.sdf_ref import sdf_ref  # noqa: E402


def legs_for(w, call):
    """kernel / graph_bwd legs of call(w) -> (dist, ...)"""
    p_leaf = w.p.detach().clone().requires_grad_()

    def kernel():
        with torch.no_grad():
            call(w)

    def graph_bwd():
        p0 = w.p
        w.p = p_leaf
        try:
            call(w)[0].sum().backward()
        finally:
            w.p = p0
    return {"kernel": kernel, "graph_bwd": graph_bwd}


def brute_nearest(w, md):
    """nearest body of every ball of a circle world (obstacles included) with dense torch ops"""
    c, r = w.p[:, :w.nb, 1:], w.rad
    d = (c.unsqueeze(2) - c.unsqueeze(1)).norm(dim=3) - r.unsqueeze(2) - r.unsqueeze(1)
    d = d + torch.diag(torch.full((w.nb,), math.inf, dtype=d.dtype, device=d.device))
    if w.no:
        s = torch.stack([sdf_ref(None, None, None, w.ov[:, k:k + 1], c, md, chunk=64)[0] for k in range(w.no)], 2)
        d = torch.cat([d, s - r.unsqueeze(2)], 2)
    best, body = d.min(2)
    return torch.where(best <= md, best, torch.full_like(best, md)), torch.where(best <= md, body, -1)


def check_brute(w, md):
    with torch.no_grad():
        d, body, _, _, _ = w.nearest(torch.arange(w.nb), md)
        bd, bb = brute_nearest(w, md)
    assert float((d - bd).abs().max()) < 1e-9, float((d - bd).abs().max())
    return float((body == bb).double().mean())


def hull_world(B, n=16, V=8, seed=0):
    """n hulls of V vertices per scene on a 4 x 4 grid (radius 4..9, spacing 25), over a floor"""
    g = torch.Generator().manual_seed(seed)
    k = torch.arange(n)
    centre = torch.stack([25.0 * (k % 4), 25.0 * (k // 4)], 1).double() + 3 * torch.rand(B, n, 2, generator=g).double()
    ang = torch.sort(2 * math.pi * torch.rand(B, n, V, generator=g, dtype=torch.float64), 2).values
    rr = (4 + 5 * torch.rand(B, n, 1, generator=g, dtype=torch.float64)).unsqueeze(3)
    pv = centre.unsqueeze(2) + rr * torch.stack([torch.cos(ang), torch.sin(ang)], 3)
    floor = rect_vertices([37.5, 100.0], [200.0, 20.0]).unsqueeze(0)
    return BatchedWorld(torch.zeros(B, 0, 2, dtype=torch.float64), torch.zeros(B, 0, dtype=torch.float64),
                        polygons=pv, obstacles=floor, gravity=G, strict_no_penetration=False, device="cuda")


def gon_world(B, V=256, gap=2.0):
    """two regular V-gons of radius 10 per scene, rotated apart, gap apart (negative: overlapping)"""
    a = 2 * math.pi * torch.arange(V, dtype=torch.float64) / V
    ring = 10.0 * torch.stack([torch.cos(a), torch.sin(a)], 1)
    tilt = 2 * math.pi * torch.rand(B, 1, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    rot = torch.stack([torch.cos(a + tilt) * 10.0, torch.sin(a + tilt) * 10.0], 2)
    pv = torch.stack([ring.expand(B, V, 2), rot + torch.tensor([20.0 + gap, 0.0], dtype=torch.float64)], 1)
    return BatchedWorld(torch.zeros(B, 0, 2, dtype=torch.float64), torch.zeros(B, 0, dtype=torch.float64),
                        polygons=pv, gravity=None, strict_no_penetration=False, device="cuda")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=1024)
    args = ap.parse_args()
    B = args.batch
    md = 1000.0
    # (a)
    ic = make_ball_pile(B, nballs=24, cols=6, seed=2000, gap=0.05)
    w = BatchedWorld(gravity=G, dt=1.0 / 30, obstacles=bin_obstacles(ic), **balls(ic))
    w.step()
    q = torch.arange(w.nb)
    agree = check_brute(w, md)
    legs = legs_for(w, lambda v: v.nearest(q, md))

    def brute():
        with torch.no_grad():
            brute_nearest(w, md)
    legs["brute"] = brute
    pairing("(a) %d piles of 24 balls in a 3-obstacle bin: nearest for all 24 balls" % B, legs, args,
            {"B": B, "K": 24, "body_agreement_with_brute": agree})
    # (b)
    wh = hull_world(256)
    hq = torch.arange(16)
    pairs = torch.triu_indices(16, 16, 1).t()
    pairing("(b) 256 scenes of 16 hulls (nv 8) and a floor: nearest for all hulls", legs_for(wh, lambda v: v.nearest(hq, md)),
            args, {"B": 256, "K": 16})
    pairing("(b) 256 scenes of 16 hulls (nv 8) and a floor: distance over all 120 hull pairs",
            legs_for(wh, lambda v: v.distance(pairs, md)), args, {"B": 256, "K": 120})
    # (c)
    for gap in (2.0, -2.0):
        wg = gon_world(256, gap=gap)
        with torch.no_grad():
            dg = wg.distance([[0, 1]], md)[0]
        pairing("(c) 256 pairs of 256-gons, %s" % ("separated" if gap > 0 else "overlapping"),
                legs_for(wg, lambda v: v.distance([[0, 1]], md)), args,
                {"B": 256, "K": 1, "dist_mean": float(dg.mean())})
    # (d)
    ic1 = make_ball_pile(1, nballs=512, cols=32, seed=0)
    w1 = BatchedWorld(ic1["pos"], ic1["rad"], vel=ic1["vel"], mass=ic1["mass"], restitution=ic1["rest"],
                      fric_coeff=ic1["fric"], gravity=G, static=[0], dt=1.0 / 30)
    agree1 = check_brute(w1, md)
    q1 = torch.arange(w1.nb)
    legs = legs_for(w1, lambda v: v.nearest(q1, md))

    def brute1():
        with torch.no_grad():
            brute_nearest(w1, md)
    legs["brute"] = brute1
    pairing("(d) one 512-ball pile: nearest for all balls", legs, args,
            {"B": 1, "K": int(w1.nb), "body_agreement_with_brute": agree1})
    # (e)
    wc = BatchedWorld(gravity=G, dt=1.0 / 30, obstacles=bin_obstacles(ic), **balls(ic))

    def nearest():
        with torch.no_grad():
            wc.nearest(q, md)

    def step():
        with torch.no_grad():
            wc.step()
    out = pairing("(e) one nearest (24 balls) vs one step(), %d piles of 24 balls" % B,
                  {"nearest": nearest, "step": step}, args, {"B": B})
    print(json.dumps({"nearest_over_step": out["nearest"]["ms_median"] / out["step"]["ms_median"]}), flush=True)


if __name__ == "__main__":
    main()
