"""World-steps per second of `BatchedWorld` with a static `Rect` floor obstacle against the same piles on the pinned
floor ball of `bench.py --config world`, and of a 512-ball pile in a bin (floor + two walls, banded kernel) against
the same pile on a pinned floor ball (config 4's scene). Runs of the two legs of a pairing alternate; prints one
JSON line per pairing with the median and the spread (min, max) of every leg, plus the card and its power limit.

    python scripts/obstacle_bench.py [--rounds 5] [--steps 10] [--warmup 3] [--batch 1024]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lcp_physics_b200.scenes import make_ball_pile  # noqa: E402
from lcp_physics_b200.world import BatchedWorld, rect_vertices  # noqa: E402


def card():
    """Name and power limit of the device in use, queried by its UUID (CUDA_VISIBLE_DEVICES renumbers devices)."""
    dev = torch.cuda.current_device()
    name = torch.cuda.get_device_name(dev)
    uuid = getattr(torch.cuda.get_device_properties(dev), "uuid", None)
    if uuid is None:
        return name + " (power limit not read: no device UUID)"
    uuid = str(uuid)
    uuid = uuid if uuid.startswith(("GPU-", "MIG-")) else "GPU-" + uuid
    try:
        out = subprocess.run(["nvidia-smi", "--id=" + uuid, "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or name + " (power limit not read)"
    except (OSError, subprocess.SubprocessError):
        return name + " (power limit not read)"


def pinned_world(ic):
    return BatchedWorld(ic["pos"], ic["rad"], vel=ic["vel"], mass=ic["mass"], restitution=ic["rest"],
                        fric_coeff=ic["fric"], gravity=100.0, static=[0], dt=1.0 / 30)


def obstacle_world(ic, walls):
    """The same balls without the floor ball (body 0); a Rect floor whose top is the floor ball's top (y = 500)."""
    x = ic["pos"][0, 1:, 0]
    lo, hi = float(x.min()) - 10.0, float(x.max()) + 10.0
    obst = [rect_vertices([0.5 * (lo + hi), 510.0], [hi - lo + 200.0, 20.0])]
    if walls:
        obst += [rect_vertices([lo - 10.0 - 1.0, 300.0], [20.0, 398.0]), rect_vertices([hi + 10.0 + 1.0, 300.0], [20.0, 398.0])]
    return BatchedWorld(ic["pos"][:, 1:], ic["rad"][:, 1:], vel=ic["vel"][:, 1:], mass=ic["mass"][:, 1:],
                        restitution=ic["rest"][:, 1:], fric_coeff=ic["fric"][:, 1:], gravity=100.0, dt=1.0 / 30,
                        obstacles=torch.stack(obst), obstacle_fric=0.9, obstacle_rest=0.5)


def rate(make, B, steps, warmup):
    w = make()
    for _ in range(warmup):
        w.step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        w.step()
    e1.record()
    torch.cuda.synchronize()
    return B * steps / (e0.elapsed_time(e1) * 1e-3), float(w.counts.float().mean())


def pairing(name, legs, B, args):
    res = {k: [] for k in legs}
    ncs = {}
    for _ in range(args.rounds):
        for k, mk in legs.items():                       # alternate the legs inside every round
            r, nc = rate(mk, B, args.steps, args.warmup)
            res[k].append(r)
            ncs[k] = nc
    out = {"pairing": name, "unit": "world-steps/s", "card": card(), "rounds": args.rounds, "steps": args.steps, "B": B}
    for k, v in res.items():
        out[k] = {"median": statistics.median(v), "min": min(v), "max": max(v), "mean_contacts_per_world": ncs[k]}
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=1024)
    args = ap.parse_args()
    ic = make_ball_pile(args.batch, nballs=24, cols=6, seed=2000, gap=0.05)
    pairing("1024 piles of 24 balls: Rect floor obstacle vs pinned floor ball",
            {"obstacle_floor": lambda: obstacle_world(ic, False), "pinned_floor_ball": lambda: pinned_world(ic)},
            args.batch, args)
    big = make_ball_pile(1, nballs=512, cols=32, seed=0)
    pairing("one 512-ball pile (banded kernel): bin of 3 obstacles vs pinned floor ball",
            {"obstacle_bin": lambda: obstacle_world(big, True), "pinned_floor_ball": lambda: pinned_world(big)}, 1, args)


if __name__ == "__main__":
    main()
