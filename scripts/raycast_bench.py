"""Ray casts against `BatchedWorld` scenes (lcpb200_raycast, `raycast`, `lidar`), timed on the GPU.

* (a) 1024 piles of 24 balls in a bin of 3 obstacles, 64 lidar rays per scene from ball 0:
    kernel   `lidar` with nothing differentiated (the kernel's distances and normals);
    graph    `lidar` with the state requiring grad (the kernel's choices, then the torch mirror);
    ray_ref  the dense brute force of tests/ray_ref.py on the same GPU;
* (b) one 512-ball pile (BASELINE config 4) with 4096 rays from its centre: kernel and graph;
* (c) one `lidar` call against one `step()` of the worlds in (a).
Legs of a pairing alternate inside every round; prints one JSON line per pairing with the median and the spread
(min, max) of every leg, and the card and its power limit read in the same run.

    python scripts/raycast_bench.py [--rounds 5] [--calls 20] [--warmup 3] [--batch 1024]
"""
import argparse
import json
import math
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lcp_physics_b200.scenes import make_ball_pile  # noqa: E402
from lcp_physics_b200.world import BatchedWorld  # noqa: E402
from scripts.hetero_bench import G, balls, bin_obstacles  # noqa: E402
from scripts.obstacle_bench import card  # noqa: E402
from tests.ray_ref import ray_ref  # noqa: E402


def timed(fn, calls, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / calls


def pairing(name, legs, args, extra=None):
    res = {k: [] for k in legs}
    for _ in range(args.rounds):
        for k, fn in legs.items():                       # alternate the legs inside every round
            res[k].append(timed(fn, args.calls, args.warmup))
    out = {"pairing": name, "card": card(), "rounds": args.rounds, "calls": args.calls}
    out.update(extra or {})
    for k, v in res.items():
        out[k] = {"ms_median": statistics.median(v), "ms_min": min(v), "ms_max": max(v)}
    print(json.dumps(out), flush=True)
    return out


def legs_for(w, mount, n_rays, max_dist, with_ref=True):
    """kernel / graph / ray_ref legs of `lidar(mount, n_rays, max_dist)` on world w"""
    p_leaf = w.p.detach().clone().requires_grad_()

    def kernel():
        with torch.no_grad():
            w.lidar(mount, n_rays, max_dist)

    def graph():
        p0 = w.p
        w.p = p_leaf
        try:
            w.lidar(mount, n_rays, max_dist)
        finally:
            w.p = p0

    k = torch.arange(n_rays, dtype=w.dtype, device=w.device)
    ang = w.p[:, mount, 0:1].detach() + k * (2 * math.pi / n_rays)
    u = torch.stack([torch.cos(ang), torch.sin(ang)], 2)
    o = w.p[:, mount, 1:].detach().unsqueeze(1).expand(-1, n_rays, -1)
    ov = w.ov if w.no else None

    def ref():
        with torch.no_grad():
            ray_ref(w.p[:, :w.nb, 1:], w.rad, None, ov, o, u, max_dist, chunk=64)
    legs = {"kernel": kernel, "graph": graph}
    if with_ref:
        legs["ray_ref"] = ref
    return legs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=1024)
    args = ap.parse_args()
    B = args.batch
    ic = make_ball_pile(B, nballs=24, cols=6, seed=2000, gap=0.05)
    w = BatchedWorld(gravity=G, dt=1.0 / 30, obstacles=bin_obstacles(ic), **balls(ic))
    w.step()                                              # a settled-in state, contacts and all
    # (a) the readings agree before they are timed
    with torch.no_grad():
        dk, bk, _ = w.lidar(0, 64, 400.0)
    leg = legs_for(w, 0, 64, 400.0)
    p_leaf = w.p.detach().clone().requires_grad_()
    p0, w.p = w.p, p_leaf
    dg, bg, _ = w.lidar(0, 64, 400.0)
    w.p = p0
    assert torch.equal(bk, bg) and float((dk - dg.detach()).abs().max()) < 1e-9
    pairing("(a) lidar, %d piles of 24 balls in a 3-obstacle bin, 64 rays per scene" % B, leg, args,
            {"B": B, "rays_per_scene": 64, "hit_fraction": float((bk >= 0).float().mean())})
    # (b) one 512-ball pile, 4096 rays from the pile's centre ball
    ic1 = make_ball_pile(1, nballs=512, cols=32, seed=0)
    w1 = BatchedWorld(ic1["pos"], ic1["rad"], vel=ic1["vel"], mass=ic1["mass"], restitution=ic1["rest"],
                      fric_coeff=ic1["fric"], gravity=G, static=[0], dt=1.0 / 30)
    mid = int(((w1.p[0, 1:, 1:] - w1.p[0, 1:, 1:].mean(0)).norm(dim=1)).argmin()) + 1
    pairing("(b) 4096 rays in one 512-ball pile", legs_for(w1, mid, 4096, 1000.0), args, {"B": 1, "rays": 4096})
    # (c) one lidar call against one step of the worlds in (a)
    wc = BatchedWorld(gravity=G, dt=1.0 / 30, obstacles=bin_obstacles(ic), **balls(ic))

    def lidar():
        with torch.no_grad():
            wc.lidar(0, 64, 400.0)

    def step():
        with torch.no_grad():
            wc.step()
    out = pairing("(c) one lidar call (64 rays) vs one step(), %d piles of 24 balls" % B,
                  {"lidar": lidar, "step": step}, args, {"B": B})
    print(json.dumps({"lidar_over_step": out["lidar"]["ms_median"] / out["step"]["ms_median"]}), flush=True)


if __name__ == "__main__":
    main()
