"""World-steps per second of `BatchedWorld` with constraints, and the cost of the no-contact mask in the contact walk:
  1. 1024 chain_demo worlds (10 Rect links: XConstraint + YConstraint on the top link, 9 Joints, no_contact between
     neighbours, Gravity on links 1-9, a projectile circle under a horizontal impulse for t < 0.1, post-stabilisation),
     in fp64 and in fp32;
  2. the contact walk with geometry of those worlds: lcpb200_contacts with no_contact (the 9 neighbour pairs
     excluded) against lcpb200_contacts without it (no pair excluded) on the same bodies.
Legs of a pairing alternate inside every round; prints one JSON line per pairing with the median and the spread
(min, max) of every leg, plus the card and its power limit.

    python scripts/joint_bench.py [--rounds 5] [--steps 10] [--warmup 3] [--batch 1024]
"""
import argparse
import ctypes
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lcp_physics_b200 import _lib  # noqa: E402
from lcp_physics_b200.world import BatchedWorld, Joint, XConstraint, YConstraint, rect_vertices  # noqa: E402
from scripts.polygon_bench import rate, report  # noqa: E402

f64 = torch.float64


def chain_world(B, dtype, seed=0):
    """chain_demo (demos/demo.py) with the projectile 100 px from the chain; per-world jitter of its height"""
    g = torch.Generator().manual_seed(seed)
    links = torch.stack([rect_vertices([300.0, 50.0 + 50.0 * i], [20.0, 60.0]) for i in range(10)])
    cons = [XConstraint(1), YConstraint(1)] + [Joint(1 + i, i, [300.0, 25.0 + 50.0 * i]) for i in range(1, 10)]
    pos = torch.stack([torch.full((B,), 200.0, dtype=f64), 500.0 + 20.0 * (torch.rand(B, generator=g, dtype=f64) - 0.5)],
                      1).unsqueeze(1)

    def push(t):
        f = torch.zeros(B, 11, 3, dtype=t.dtype, device=t.device)
        f[:, 0, 1] = torch.where(t < 0.1, torch.full_like(t, 2000.0), torch.zeros_like(t))
        return f
    return BatchedWorld(pos.to(dtype), 20.0, restitution=0.9, gravity=100.0, gravity_mask=[False, False] + [True] * 9,
                        dt=1.0 / 30, post_stab=True, polygons=links.unsqueeze(0).expand(B, -1, -1, -1), poly_rest=0.9,
                        constraints=cons, no_contact=[(1 + i, i) for i in range(1, 10)], external_force=push,
                        device="cuda")


def walk_time(w, masked, reps=50):
    """ms per call of the contact walk with geometry on w's bodies, with or without w's no-contact mask"""
    lib, B, cap, dev = _lib.load(), w.B, w.cap, w.device
    i32 = lambda *s: torch.empty(*s, dtype=torch.int32, device=dev)
    b1, b2, feat, counts = i32(B, cap), i32(B, cap), i32(B, cap), i32(B)
    geo = [torch.empty(B, cap, *s, dtype=w.dtype, device=dev) for s in ((2,), (2,), (2,), (), (), ())]
    st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    pv, pcen = w.polygon_vertices().contiguous(), w.p[:, w.nb:, 1:].contiguous()
    ins = [t.contiguous() for t in (w.p[:, :w.nb, 1:], w.rad, w.fric_coeff, w.restitution, pv, pcen, w.pfric, w.prest)]
    args = [_lib.dtype_code(w.dtype), B, w.nb, w.np, w.no, w.nv, cap, w.eps, *[_lib.ptr(t) for t in ins],
            None, None, None, None, *[_lib.ptr(t) for t in (b1, b2, counts, feat)], *[_lib.ptr(t) for t in geo]]
    call = lambda: lib.lcpb200_contacts(*args, _lib.ptr(w.nc_mask) if masked else None, st)
    for _ in range(5):
        _lib.check(call())
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        _lib.check(call())
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=1024)
    args = ap.parse_args()
    _lib.require_cuda()
    res = {"chain_fp64": [], "chain_fp32": []}
    info = {}
    for _ in range(args.rounds):
        for k, dt in (("chain_fp64", f64), ("chain_fp32", torch.float32)):
            r, nc, big = rate(lambda: chain_world(args.batch, dt), args.batch, args.steps, args.warmup)
            res[k].append(r)
            info[k] = {"mean_contacts_per_world": nc, "banded_kernel": big}
    report("BatchedWorld chain_demo (10 links, 9 joints + X and Y constraints)", "world-steps/s", res,
           {"steps": args.steps, "warmup": args.warmup, "batch": args.batch, "legs": info}, args)
    w = chain_world(args.batch, f64)
    for _ in range(12):                                    # the projectile reaches the chain
        w.step()
    walk = {"masked_walk_ms": [], "unmasked_walk_ms": []}
    for _ in range(args.rounds):
        walk["masked_walk_ms"].append(walk_time(w, True))
        walk["unmasked_walk_ms"].append(walk_time(w, False))
    report("contact walk + geometry, %d chain worlds of %d bodies, 9 pairs excluded" % (w.B, w.nd), "ms", walk,
           {"bodies": w.nd}, args)


if __name__ == "__main__":
    main()
