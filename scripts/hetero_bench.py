"""Heterogeneous batches in `BatchedWorld` (per-scene active bodies), timed on the GPU.

* world-steps/s of 1024 piles of 8-24 balls (a random count per scene) in a bin of 3 obstacles:
    hetero   one batch of 24-ball worlds, each scene's first k balls active (`active=`);
    grouped  the same scenes as one homogeneous world per ball count, every group stepped once per step;
    parked   one batch of 24-ball worlds whose unused balls are parked far apart, their gravity cancelled by
             `external_force` (the workaround without `active`);
* the contact walk alone (`find_contacts`: walk + geometry kernel) on 1024 scenes of 96 scattered balls in a bin, at
  25 % and 100 % of the balls active, against today's walk of the same world without `active`.
Legs of a pairing alternate inside every round; prints one JSON line per pairing with the median and the spread
(min, max) of every leg, and the card and its power limit read in the same run.

    python scripts/hetero_bench.py [--rounds 5] [--steps 10] [--warmup 3] [--batch 1024]
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lcp_physics_b200.scenes import make_ball_pile  # noqa: E402
from lcp_physics_b200.world import BatchedWorld, rect_vertices  # noqa: E402
from scripts.obstacle_bench import card  # noqa: E402

G = 100.0


def bin_obstacles(ic):
    x = ic["pos"][0, 1:, 0]
    lo, hi = float(x.min()) - 10.0, float(x.max()) + 10.0
    return torch.stack([rect_vertices([0.5 * (lo + hi), 510.0], [hi - lo + 200.0, 20.0]),
                        rect_vertices([lo - 11.0, 300.0], [20.0, 398.0]), rect_vertices([hi + 11.0, 300.0], [20.0, 398.0])])


def balls(ic, rows=None, k=None):
    """the pile's balls (body 0, the floor ball, dropped), scenes `rows`, the first k balls"""
    rows = slice(None) if rows is None else rows
    k = slice(1, None) if k is None else slice(1, 1 + k)
    return dict(pos=ic["pos"][rows, k], rad=ic["rad"][rows, k], vel=ic["vel"][rows, k], mass=ic["mass"][rows, k],
                restitution=ic["rest"][rows, k], fric_coeff=ic["fric"][rows, k])


def hetero_world(ic, counts):
    nb = ic["pos"].shape[1] - 1
    act = torch.arange(nb + 3).unsqueeze(0) < counts.unsqueeze(1)
    act[:, nb:] = True                                               # the bin
    return BatchedWorld(gravity=G, dt=1.0 / 30, obstacles=bin_obstacles(ic), active=act, **balls(ic))


class Grouped:
    """one homogeneous world per ball count, stepped in turn"""

    def __init__(self, ic, counts):
        self.worlds = [BatchedWorld(gravity=G, dt=1.0 / 30, obstacles=bin_obstacles(ic),
                                    **balls(ic, (counts == k).nonzero()[:, 0], k))
                       for k in sorted(set(counts.tolist()))]
        self.counts = torch.cat([w.counts for w in self.worlds])

    def step(self):
        for w in self.worlds:
            w.step()
        self.counts = torch.cat([w.counts for w in self.worlds])


def parked_world(ic, counts):
    """unused balls parked 100 apart at x = 1e5, their gravity cancelled by an external force"""
    B, nb = ic["pos"].shape[0], ic["pos"].shape[1] - 1
    b = balls(ic)
    park = torch.arange(nb).unsqueeze(0) >= counts.unsqueeze(1)      # [B, nb]
    pos = b["pos"].clone()
    pos[..., 0] = torch.where(park, 1.0e5 + 100.0 * torch.arange(nb, dtype=pos.dtype), pos[..., 0])
    b["pos"] = pos
    w = BatchedWorld(gravity=G, dt=1.0 / 30, obstacles=bin_obstacles(ic), **b)
    f = torch.zeros(B, nb, 3, dtype=pos.dtype, device=w.device)
    f[..., 2] = -w.fext[:, 2::3] * park.to(w.device)
    w.external_force = lambda t: f
    return w


def timed(w, steps, warmup, B, call="step"):
    fn = getattr(w, call)
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, float(w.counts.float().mean())


def pairing(name, legs, args, B, call="step"):
    res = {k: [] for k in legs}
    ncs = {}
    for _ in range(args.rounds):
        for k, mk in legs.items():                       # alternate the legs inside every round
            ms, nc = timed(mk(), args.steps, args.warmup, B, call)
            res[k].append(ms)
            ncs[k] = nc
    out = {"pairing": name, "card": card(), "rounds": args.rounds, "steps": args.steps, "B": B}
    for k, v in res.items():
        rate = [B / (m * 1e-3) for m in v]
        out[k] = {"ms_median": statistics.median(v), "ms_min": min(v), "ms_max": max(v),
                  "world_steps_per_s_median": statistics.median(rate), "mean_contacts_per_scene": ncs[k]}
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=1024)
    args = ap.parse_args()
    B = args.batch
    ic = make_ball_pile(B, nballs=24, cols=6, seed=2000, gap=0.05)
    counts = torch.randint(8, 25, (B,), generator=torch.Generator().manual_seed(1))
    pairing("%d piles of 8-24 balls in a bin: one heterogeneous batch vs homogeneous batches per count vs parked "
            "balls" % B, {"hetero": lambda: hetero_world(ic, counts), "grouped": lambda: Grouped(ic, counts),
                          "parked": lambda: parked_world(ic, counts)}, args, B)
    # the walk alone: 96 balls scattered in a 400 x 300 box (no start check), 25 % / 100 % active, and today's walk
    g = torch.Generator().manual_seed(3)
    nb = 96
    pos = torch.rand(B, nb, 2, generator=g, dtype=torch.float64) * torch.tensor([400.0, 300.0], dtype=torch.float64)
    obst = torch.stack([rect_vertices([200.0, 320.0], [440.0, 20.0]), rect_vertices([-20.0, 150.0], [20.0, 340.0]),
                        rect_vertices([420.0, 150.0], [20.0, 340.0])])
    quarter = torch.rand(B, nb + 3, generator=g) < 0.25
    quarter[:, nb:] = True
    walk = lambda act: BatchedWorld(pos, 6.0, obstacles=obst, active=act, strict_no_penetration=False,
                                    contact_capacity=512)
    with torch.no_grad():
        pairing("the contact walk alone (find_contacts), %d scenes of %d balls in a bin" % (B, nb),
                {"active_25pct": lambda: walk(quarter), "active_100pct": lambda: walk(True),
                 "no_active_argument": lambda: walk(None)}, args, B, call="find_contacts")


if __name__ == "__main__":
    main()
