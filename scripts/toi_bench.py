"""Times of impact of `BatchedWorld` bodies (lcpb200_time_of_impact, `first_impact`) and the continuous-collision
step (`ccd=True`), timed on the GPU.

* (a) 1024 piles of 24 balls in a bin of 3 obstacles: `first_impact` of every ball by v dt;
* (b) 256 scenes of 16 spinning hulls (8 vertices) over a floor: `first_impact` of every hull by 10 v dt, with up to
  1 radian of rotation;
* (c) the worlds of (a): one `step()` with ccd off and with ccd on.
Each has a kernel leg (nothing differentiated) and a graph_bwd leg (the state requiring grad, then a backward pass of
the first output's sum; for (c) of the positions after the step). Legs of a pairing alternate inside every round;
prints one JSON line per pairing with the median and the spread (min, max) of every leg, and the card and its power
limit read in the same run.

    python scripts/toi_bench.py [--rounds 5] [--calls 20] [--warmup 3] [--batch 1024]
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lcp_physics_b200.scenes import make_ball_pile  # noqa: E402
from lcp_physics_b200.world import BatchedWorld  # noqa: E402
from scripts.distance_bench import hull_world, legs_for  # noqa: E402
from scripts.hetero_bench import G, balls, bin_obstacles  # noqa: E402
from scripts.raycast_bench import pairing  # noqa: E402


def motion_of(w, scale=1.0):
    """each dynamic body's motion over `scale` steps, v dt"""
    return (w.v.reshape(w.B, w.nd, 3) * (w.dt * scale)).detach().contiguous()


def step_legs(w):
    """kernel / graph_bwd legs of one step() from a fixed state"""
    p0, v0, t0 = w.p.detach().clone(), w.v.detach().clone(), w.t.clone()

    def reset(p):
        w.p, w.v, w.t = p, v0.clone(), t0.clone()
        w.find_contacts()

    def kernel():
        with torch.no_grad():
            reset(p0.clone())
            w.step()

    def graph_bwd():
        reset(p0.clone().requires_grad_())
        w.step()
        w.p.sum().backward()
    return {"kernel": kernel, "graph_bwd": graph_bwd}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=1024)
    args = ap.parse_args()
    B = args.batch
    # (a)
    ic = make_ball_pile(B, nballs=24, cols=6, seed=2000, gap=0.05)
    w = BatchedWorld(gravity=G, dt=1.0 / 30, obstacles=bin_obstacles(ic), **balls(ic))
    for _ in range(3):
        w.step()
    q = torch.arange(w.nd)
    m = motion_of(w)
    with torch.no_grad():
        hits = float((w.first_impact(q, m, gap=w.eps / 2, skip=w.eps)[1] >= 0).double().mean())
    pairing("(a) %d piles of 24 balls in a 3-obstacle bin: first_impact of every ball by v dt" % B,
            legs_for(w, lambda v: v.first_impact(q, m, gap=v.eps / 2, skip=v.eps)), args,
            {"B": B, "K": 24, "hit_fraction": hits})
    # (b)
    wh = hull_world(256)
    wh.step()
    g = torch.Generator().manual_seed(5)
    mh = motion_of(wh, 10.0)
    mh[..., 0] = (2 * torch.rand(256, 16, generator=g, dtype=torch.float64) - 1).cuda()
    hq = torch.arange(16)
    with torch.no_grad():
        hits = float((wh.first_impact(hq, mh)[1] >= 0).double().mean())
    pairing("(b) 256 scenes of 16 spinning hulls (nv 8) and a floor: first_impact of every hull by 10 v dt",
            legs_for(wh, lambda v: v.first_impact(hq, mh)), args, {"B": 256, "K": 16, "hit_fraction": hits})
    # (c)
    legs = {}
    for ccd in (False, True):
        ws = BatchedWorld(gravity=G, dt=1.0 / 30, obstacles=bin_obstacles(ic), ccd=ccd, **balls(ic))
        for _ in range(3):
            ws.step()
        for k, fn in step_legs(ws).items():
            legs[("ccd_" if ccd else "discrete_") + k] = fn
    pairing("(c) %d piles of 24 balls: one step() with ccd off and on" % B, legs, args, {"B": B})


if __name__ == "__main__":
    main()
