"""World-steps per second of `BatchedWorld` with dynamic polygons, and the time of its contact walk:
  1. 1024 worlds of 12 boxes + 12 circles in a bin of 3 obstacles (condensed kernels, fp64);
  2. one large mixed bin, 80 boxes + 16 hulls + 24 circles (3 * 120 > 128: banded kernel);
  3. the contact walk (lcpb200_contacts with feat: the polygon walk, detection + geometry) of pairing 1's worlds against
     the circle-only walk (lcpb200_contacts without feat) over the same number of bodies, all of them circles.
Legs of a pairing alternate inside every round; prints one JSON line per pairing with the median and the spread
(min, max) of every leg, plus the card and its power limit.

    python scripts/polygon_bench.py [--rounds 5] [--steps 10] [--warmup 3] [--batch 1024]
"""
import argparse
import ctypes
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lcp_physics_b200 import _lib  # noqa: E402
from lcp_physics_b200.world import BatchedWorld, rect_vertices  # noqa: E402
from scripts.obstacle_bench import card  # noqa: E402

f64 = torch.float64


def bin_world(B, cols, rows, ncirc, seed, hull_every=0):
    """rows x cols boxes (30 x 16) resting on each other in a bin (every `hull_every`-th a hexagon), circles (r 6) on
    top; per-world jitter of rotation and position"""
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *s: torch.rand(*s, generator=g, dtype=f64)
    base = lambda row: 500.0 - 16.06 * row - 0.03
    polys = []
    for k in range(rows * cols):
        cx, row = 100.0 + 34.0 * (k % cols), k // cols
        if hull_every and k % hull_every == hull_every - 1:
            t = torch.arange(6, dtype=f64) * (3.14159265358979 / 3)
            v = torch.stack([cx + 9.0 * torch.cos(t), base(row) - 8.0 + 8.0 * torch.sin(t)], 1)
        else:
            v = rect_vertices([cx, base(row) - 8.0], [30.0, 16.0], 0.0)
            v = torch.cat([v, v[3:].expand(2, 2)])
        polys.append(v)
    pv = torch.stack(polys).unsqueeze(0).repeat(B, 1, 1, 1)
    pv[..., 0] += 0.5 * (rnd(B, rows * cols, 1) - 0.5)
    top = base(rows) - 6.0 - 0.03
    pos = torch.stack([100.0 + 34.0 * cols / ncirc * torch.arange(ncirc, dtype=f64).expand(B, -1) + rnd(B, ncirc),
                       top - 0.04 * rnd(B, ncirc)], 2)
    w = 34.0 * cols + 80.0
    obst = torch.stack([rect_vertices([80.0 + w / 2 - 40.0, 510.0], [w + 40.0, 20.0]),
                        rect_vertices([60.0, 400.0], [20.0, 220.0]), rect_vertices([100.0 + 34.0 * cols + 3.0, 400.0],
                                                                                   [20.0, 220.0])])
    obst = torch.cat([obst, obst[:, 3:].expand(-1, 2, -1)], 1)
    return dict(pos=pos, polys=pv, obst=obst)


def make_world(sc):
    return BatchedWorld(sc["pos"], 6.0, gravity=100.0, dt=1.0 / 30, polygons=sc["polys"], obstacles=sc["obst"],
                        obstacle_fric=0.6, obstacle_rest=0.3, poly_fric=0.5, poly_rest=0.3, fric_coeff=0.5,
                        restitution=0.3, device="cuda")


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
    return B * steps / (e0.elapsed_time(e1) * 1e-3), float(w.counts.float().mean()), w.large


def walk_time(w, circles_only, reps=50):
    """ms per call of the contact walk with geometry: w's own walk, or the circle-only walk over as many circles"""
    lib, B, cap, dev = _lib.load(), w.B, w.cap, w.device
    i32 = lambda *s: torch.empty(*s, dtype=torch.int32, device=dev)
    b1, b2, feat, counts = i32(B, cap), i32(B, cap), i32(B, cap), i32(B)
    geo = [torch.empty(B, cap, *s, dtype=f64, device=dev) for s in ((2,), (2,), (2,), (), (), ())]
    st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    if circles_only:                                       # every dynamic body a circle at its centre
        pos = w.p[:, :, 1:].contiguous()
        rad = torch.full((B, w.nd), 8.0, dtype=f64, device=dev)
        mat = torch.full((B, w.nd), 0.5, dtype=f64, device=dev)
        args = (_lib.dtype_code(f64), B, w.nd, 0, w.no, w.nv, cap, w.eps,
                *[_lib.ptr(t) for t in (pos, rad, mat, mat, None, None, None, None, w.ov, w.oref, w.ofric, w.orest,
                                        b1, b2, counts, None)],
                *[_lib.ptr(t) for t in geo], None, st)
    else:
        pv, pcen = w.polygon_vertices().contiguous(), w.p[:, w.nb:, 1:].contiguous()
        ins = [t.contiguous() for t in (w.p[:, :w.nb, 1:], w.rad, w.fric_coeff, w.restitution, pv, pcen, w.pfric,
                                        w.prest, w.ov, w.oref, w.ofric, w.orest)]         # held for every call
        args = (_lib.dtype_code(f64), B, w.nb, w.np, w.no, w.nv, cap, w.eps, *[_lib.ptr(t) for t in ins],
                *[_lib.ptr(t) for t in (b1, b2, counts, feat)], *[_lib.ptr(t) for t in geo], None, st)
    call = lambda: lib.lcpb200_contacts(*args)
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


def report(name, unit, res, extra, args):
    out = {"pairing": name, "unit": unit, "card": card(), "rounds": args.rounds}
    out.update(extra)
    for k, v in res.items():
        out[k] = {"median": statistics.median(v), "min": min(v), "max": max(v)}
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=1024)
    args = ap.parse_args()
    small = bin_world(args.batch, 6, 2, 12, seed=1)
    large = bin_world(1, 12, 8, 24, seed=2, hull_every=6)
    res = {"boxes_and_circles_1024": [], "large_mixed_bin": []}
    info = {}
    for _ in range(args.rounds):
        for k, (sc, B) in (("boxes_and_circles_1024", (small, args.batch)), ("large_mixed_bin", (large, 1))):
            r, nc, big = rate(lambda: make_world(sc), B, args.steps, args.warmup)
            res[k].append(r)
            info[k] = {"mean_contacts_per_world": nc, "banded_kernel": big}
    report("BatchedWorld with dynamic polygons", "world-steps/s", res, {"steps": args.steps, "legs": info}, args)
    w = make_world(small)
    walk = {"polygon_walk_ms": [], "circle_only_walk_ms": []}
    for _ in range(args.rounds):
        walk["polygon_walk_ms"].append(walk_time(w, False))
        walk["circle_only_walk_ms"].append(walk_time(w, True))
    report("contact walk + geometry, %d worlds of %d dynamic bodies and 3 obstacles" % (w.B, w.nd), "ms", walk,
           {"bodies": w.nd}, args)


if __name__ == "__main__":
    main()
