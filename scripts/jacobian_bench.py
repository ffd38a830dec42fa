"""Cost of step Jacobians: batched cotangents through the engine solve against one cotangent at a time.

Scenes: 1024 piles of 24 balls on a pinned floor ball (`bench.py --config world`), 1024 chain_demo worlds (10 Rect
links, 9 joints, X and Y constraints, post-stabilisation) and one 60-ball pile (banded kernel). For each scene:
  (a) kernel: one lcpb200_engine_backward_batched call with R = 2n cotangents against R lcpb200_engine_backward calls,
      on the same saved solve of the scene's contact list (outputs preallocated for both legs);
  (b) BatchedWorld.linearize() against R sequential torch.autograd.grad calls through one autograd step.
R = 2n: one cotangent per row of the step Jacobian. Legs of a pairing alternate inside every round (CUDA events);
prints one JSON line per scene and pairing with the median and the spread (min, max) of every leg, plus the card and
its power limit.

    python scripts/jacobian_bench.py [--rounds 3] [--batch 1024]
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lcp_physics_b200 import _lib  # noqa: E402
from lcp_physics_b200.engines import _engine_args, engine_solve  # noqa: E402
from lcp_physics_b200.scenes import make_ball_pile  # noqa: E402
from lcp_physics_b200.world import BatchedWorld  # noqa: E402
from scripts.joint_bench import chain_world  # noqa: E402
from scripts.obstacle_bench import card  # noqa: E402

f64 = torch.float64


def pile_world(B, nballs, cols, seed):
    ic = make_ball_pile(B, nballs=nballs, cols=cols, seed=seed, gap=0.05)
    return BatchedWorld(ic["pos"], ic["rad"], vel=ic["vel"], mass=ic["mass"], restitution=ic["rest"],
                        fric_coeff=ic["fric"], gravity=100.0, static=[0], dt=1.0 / 30, device="cuda")


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def kernel_legs(w, R):
    """The two legs of (a) on the saved solve of w's current contact list: callables, and the tensors their
    arguments point into (kept alive by the caller while the legs run)."""
    lib = _lib.load()
    v = w.v.detach().clone().requires_grad_(True)
    b = w.v.new_zeros(w.B, w.ne) if w.ne else None
    inputs = (w.mass, w.inertia, v, w.fext, w.c_normal, w.c_p1, w.c_p2, w.c_mu, w.c_rest)
    z, _ = engine_solve(*inputs, w.c_b1, w.c_b2, w.dt, A=w.A, b=b, mode=0, max_iter=w.max_iter,
                        exact_adjoint=w.exact_adjoint, counts=w.counts)
    hd, args, held = _engine_args(z.grad_fn.meta, z.grad_fn.saved_tensors)
    gen = torch.Generator("cuda").manual_seed(0)
    G = torch.randn((R,) + tuple(z.shape), dtype=z.dtype, device=z.device, generator=gen)
    o = lambda t: torch.zeros((R,) + tuple(t.shape), dtype=t.dtype, device=t.device)
    outs = [o(t) for t in inputs]
    outs += [o(w.A), torch.zeros(R, w.B, w.ne, dtype=z.dtype, device=z.device)] if w.ne else [None, None]
    st = _lib.stream_ptr(z.device)
    flags = 1 if w.exact_adjoint else 0

    def batched():
        _lib.check(lib.lcpb200_engine_backward_batched(hd.raw, R, *args, _lib.ptr(G), *[_lib.ptr(t) for t in outs],
                                                       flags, st))

    def sequential():
        for r in range(R):
            _lib.check(lib.lcpb200_engine_backward(hd.raw, *args, _lib.ptr(G[r]),
                                                   *[_lib.ptr(None if t is None else t[r]) for t in outs], flags, st))
    return batched, sequential, held


def autograd_rows(w):
    """R = 2n torch.autograd.grad calls through one autograd step from w's state (the world is restored)."""
    saved = dict(w.__dict__)
    joints = [None if s is None else list(s) for s in w._jstate]
    ef, n, B = w.external_force, w.n, w.B
    try:
        x = torch.cat([w.get_p(), w.v], 1).detach().clone().requires_grad_(True)
        u = x.new_zeros(B, n).requires_grad_(True)
        w.p, w.v = x[:, :n].reshape(B, w.nd, 3), x[:, n:]
        ub = u.reshape(B, w.nd, 3)
        w.external_force = (lambda t: ub) if ef is None else (lambda t: ef(t) + ub)
        w.find_contacts()
        w.step()
        out = torch.cat([w.get_p(), w.v], 1)
        for r in range(2 * n):
            torch.autograd.grad(out[:, r].sum(), (x, u), retain_graph=True)
    finally:
        w.__dict__.clear()
        w.__dict__.update(saved)
        for s, old in zip(w._jstate, joints):
            if s is not None:
                s[:] = old


def report(scene, pairing, res, extra, args):
    out = {"scene": scene, "pairing": pairing, "unit": "ms", "card": card(), "rounds": args.rounds}
    out.update(extra)
    for k, v in res.items():
        out[k] = {"median": statistics.median(v), "min": min(v), "max": max(v)}
    legs = list(res)
    out["speedup_median"] = statistics.median(res[legs[1]]) / statistics.median(res[legs[0]])
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=1024)
    args = ap.parse_args()
    _lib.require_cuda()
    scenes = [("%d piles of 24 balls" % args.batch, lambda: pile_world(args.batch, 24, 6, 2000), 2),
              ("%d chain_demo worlds" % args.batch, lambda: chain_world(args.batch, f64), 12),
              ("one 60-ball pile (banded kernel)", lambda: pile_world(1, 60, 12, 4), 2)]
    for name, make, steps in scenes:
        w = make()
        for _ in range(steps):
            w.step()
        torch.cuda.synchronize()
        R = 2 * w.n
        extra = {"B": w.B, "n": w.n, "R": R, "mean_contacts_per_world": float(w.counts.float().mean()),
                 "banded_kernel": w.large}
        batched, sequential, held = kernel_legs(w, R)
        batched()
        sequential()                                           # warm-up of both legs
        torch.cuda.synchronize()
        res = {"batched_entry_R_2n": [], "sequential_R_calls": []}
        for _ in range(args.rounds):
            res["batched_entry_R_2n"].append(timed(batched))
            res["sequential_R_calls"].append(timed(sequential))
        report(name, "(a) engine backward kernel, R = 2n cotangents", res, extra, args)
        w.linearize()
        autograd_rows(w)
        torch.cuda.synchronize()
        res = {"linearize": [], "sequential_autograd_grad": []}
        for _ in range(args.rounds):
            res["linearize"].append(timed(w.linearize))
            res["sequential_autograd_grad"].append(timed(lambda: autograd_rows(w)))
        report(name, "(b) step Jacobian", res, extra, args)
        del w
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
