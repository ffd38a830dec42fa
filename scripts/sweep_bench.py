"""Shape casts and sweeps of `BatchedWorld` bodies (lcpb200_shapecast, `shapecast`, `sweep`), timed on the GPU.

* (a) 1024 piles of 24 balls in a bin of 3 obstacles:
    `shapecast` of 64 disks (radius 2) per scene against `raycast` of the same rays (what the rounding costs);
    `sweep` of all 24 balls by v dt against `nearest` of the same balls and against one `step()`;
* (b) 256 scenes of 16 hulls (8 vertices) on a floor: `sweep` of every hull;
* (c) 256 scenes of two 256-gons: `sweep` of the first onto the second (the O(V^2) polygon pair on one thread).
Each query has a kernel leg (nothing differentiated) and a graph_bwd leg (the state requiring grad, then a backward
pass of the first output's sum). Legs of a pairing alternate inside every round; prints one JSON line per pairing
with the median and the spread (min, max) of every leg, and the card and its power limit read in the same run.

    python scripts/sweep_bench.py [--rounds 5] [--calls 20] [--warmup 3] [--batch 1024]
"""
import argparse
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lcp_physics_b200.scenes import make_ball_pile  # noqa: E402
from lcp_physics_b200.world import BatchedWorld  # noqa: E402
from scripts.distance_bench import gon_world, hull_world, legs_for  # noqa: E402
from scripts.hetero_bench import G, balls, bin_obstacles  # noqa: E402
from scripts.raycast_bench import pairing  # noqa: E402


def named(legs, prefix):
    return {prefix + "_" + k: v for k, v in legs.items()}


def disp_of(w, ks):
    """each body's translation over one step, v dt"""
    return (w.v.reshape(w.B, w.nd, 3)[:, ks, 1:] * w.dt).detach().contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=1024)
    args = ap.parse_args()
    B = args.batch
    md = 200.0
    # (a)
    ic = make_ball_pile(B, nballs=24, cols=6, seed=2000, gap=0.05)
    w = BatchedWorld(gravity=G, dt=1.0 / 30, obstacles=bin_obstacles(ic), **balls(ic))
    for _ in range(3):
        w.step()
    g = torch.Generator().manual_seed(3)
    lo, hi = w.p[:, :, 1:].detach().amin((0, 1)).cpu(), w.p[:, :, 1:].detach().amax((0, 1)).cpu()
    o = (lo + (hi - lo) * torch.rand(B, 64, 2, generator=g, dtype=torch.float64)).cuda()
    a = 2 * math.pi * torch.rand(B, 64, generator=g, dtype=torch.float64)
    u = torch.stack([a.cos(), a.sin()], 2).cuda()
    with torch.no_grad():
        hits = float((w.shapecast(o, u, 2.0, md)[1] >= 0).double().mean())
    legs = named(legs_for(w, lambda v: v.shapecast(o, u, 2.0, md)), "shapecast")
    legs.update(named(legs_for(w, lambda v: v.raycast(o, u, md)), "raycast"))
    pairing("(a) %d piles of 24 balls in a 3-obstacle bin: shapecast (radius 2) vs raycast, 64 per scene" % B, legs,
            args, {"B": B, "K": 64, "shapecast_hit_fraction": hits})
    q = torch.arange(w.nb)
    d = disp_of(w, q)
    with torch.no_grad():
        hits = float((w.sweep(q, d)[1] >= 0).double().mean())
    legs = named(legs_for(w, lambda v: v.sweep(q, d)), "sweep")
    legs.update(named(legs_for(w, lambda v: v.nearest(q, md)), "nearest"))

    ws = BatchedWorld(gravity=G, dt=1.0 / 30, obstacles=bin_obstacles(ic), **balls(ic))   # stepped apart from w

    def step():
        with torch.no_grad():
            ws.step()
    legs["step"] = step
    out = pairing("(a) %d piles of 24 balls: sweep of every ball by v dt vs nearest vs one step()" % B, legs, args,
                  {"B": B, "K": 24, "sweep_hit_fraction": hits})
    print(json.dumps({"sweep_over_step": out["sweep_kernel"]["ms_median"] / out["step"]["ms_median"]}), flush=True)
    # (b)
    wh = hull_world(256)
    wh.step()
    hq = torch.arange(16)
    dh = disp_of(wh, hq) * 10
    pairing("(b) 256 scenes of 16 hulls (nv 8) and a floor: sweep of every hull by 10 v dt",
            legs_for(wh, lambda v: v.sweep(hq, dh)), args, {"B": 256, "K": 16})
    # (c)
    wg = gon_world(256, gap=2.0)
    dg = torch.tensor([[10.0, 0.0]], dtype=torch.float64, device="cuda")
    with torch.no_grad():
        fr = wg.sweep([0], dg)[0]
    pairing("(c) 256 pairs of 256-gons, 2 apart: sweep of one onto the other",
            legs_for(wg, lambda v: v.sweep([0], dg)), args, {"B": 256, "K": 1, "frac_mean": float(fr.mean())})


if __name__ == "__main__":
    main()
