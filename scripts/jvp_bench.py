"""Cost of forward-mode derivatives: batched tangents through the engine solve, and rollout sensitivities.

  (a) kernel, 1024 piles of 24 balls (condensed kernel): one lcpb200_engine_jvp_batched call with R tangents against
      R single-tangent calls, beside one lcpb200_engine_backward_batched call with R cotangents (R = 3 and R = n), on
      the same saved solve (outputs preallocated for every leg);
  (b) sensitivities of a 30-step rollout of those piles w.r.t. 3 per-scene parameters (friction offset, relative mass
      change, initial velocity change): forward mode (3 tangents, torch.func.jvp under vmap) against reverse mode (one
      torch.func.vjp of the rollout, then 2n one-hot cotangents of the final state under vmap: the full Jacobian of
      the final state w.r.t. the same parameters). Time and peak memory of each;
  (c) the same rollout comparison on one 60-ball pile (banded kernel).
Legs of a pairing alternate inside every round (CUDA events). One JSON line per pairing: median and spread (min,
max) of every leg, peak memory where measured, the card and its power limit.

    python scripts/jvp_bench.py [--rounds 5] [--batch 1024] [--steps 30]
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
from scripts.obstacle_bench import card  # noqa: E402

f64 = torch.float64


def pile_world(B, nballs, cols, seed, theta=None):
    """Piles on a pinned floor ball (bench.py --config world); theta [B, 3]: friction offset, relative mass change and
    initial x-velocity change of every ball."""
    ic = make_ball_pile(B, nballs=nballs, cols=cols, seed=seed, gap=0.05)
    ic = {k: v.cuda() for k, v in ic.items()}
    fric, mass, vel = ic["fric"], ic["mass"], ic["vel"]
    if theta is not None:
        fric = fric + theta[:, 0:1]
        mass = mass * (1 + theta[:, 1:2])
        vel = vel + theta[:, 2:3, None] * torch.tensor([0.0, 1.0, 0.0], dtype=f64, device="cuda")
    return BatchedWorld(ic["pos"], ic["rad"], vel=vel, mass=mass, restitution=ic["rest"], fric_coeff=fric,
                        gravity=100.0, static=[0], dt=1.0 / 30, exact_adjoint=True, device="cuda")


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def kernel_legs(w, R):
    """(a) on the saved solve of w's current contact list: batched JVP, R single-tangent JVPs, batched VJP; and the
    tensors their arguments point into (kept alive by the caller while the legs run)."""
    lib = _lib.load()
    v = w.v.detach().clone().requires_grad_(True)
    b = w.v.new_zeros(w.B, w.ne) if w.ne else None
    inputs = (w.mass, w.inertia, v, w.fext, w.c_normal, w.c_p1, w.c_p2, w.c_mu, w.c_rest)
    z, _ = engine_solve(*inputs, w.c_b1, w.c_b2, w.dt, A=w.A, b=b, mode=0, max_iter=w.max_iter, exact_adjoint=True,
                        counts=w.counts)
    hd, args, held = _engine_args(z.grad_fn.meta, z.grad_fn.saved_tensors)
    gen = torch.Generator("cuda").manual_seed(0)
    rnd = lambda t: torch.randn((R,) + tuple(t.shape), dtype=t.dtype, device=t.device, generator=gen)
    tg = [rnd(t) for t in inputs] + ([rnd(w.A), rnd(b)] if w.ne else [None] * 2)
    dz = torch.zeros((R,) + tuple(z.shape), dtype=z.dtype, device=z.device)
    G = rnd(z)
    o = lambda t: torch.zeros((R,) + tuple(t.shape), dtype=t.dtype, device=t.device)
    outs = [o(t) for t in inputs] + ([o(w.A), o(b)] if w.ne else [None] * 2)
    st = _lib.stream_ptr(z.device)

    def jvp_batched():
        _lib.check(lib.lcpb200_engine_jvp_batched(hd.raw, R, *args, *[_lib.ptr(t) for t in tg], _lib.ptr(dz), st))

    def jvp_sequential():
        for r in range(R):
            _lib.check(lib.lcpb200_engine_jvp_batched(hd.raw, 1, *args,
                                                      *[_lib.ptr(None if t is None else t[r]) for t in tg],
                                                      _lib.ptr(dz[r]), st))

    def vjp_batched():
        _lib.check(lib.lcpb200_engine_backward_batched(hd.raw, R, *args, _lib.ptr(G), *[_lib.ptr(t) for t in outs], 1,
                                                       st))
    return {"jvp_batched_one_call": jvp_batched, "jvp_R_single_calls": jvp_sequential,
            "vjp_batched_one_call": vjp_batched}, held


def rollout_legs(B, nballs, cols, seed, steps):
    """(b) / (c): d(final state)/d(theta) for theta [B, 3] by forward and by reverse mode."""
    theta = torch.zeros(B, 3, dtype=f64, device="cuda")

    def f(th):
        w = pile_world(B, nballs, cols, seed, th)
        for _ in range(steps):
            w.step()
        return torch.cat([w.get_p(), w.v], 1)

    out = {}

    def forward_mode():
        eye = torch.eye(3, dtype=f64, device="cuda").unsqueeze(1).expand(-1, B, -1)
        out["fwd"] = torch.func.vmap(lambda t: torch.func.jvp(f, (theta,), (t,))[1], randomness="same")(eye)   # [3, B, 2n]

    def reverse_mode():
        x, vjp_fn = torch.func.vjp(f, theta)
        eye = torch.eye(x.shape[1], dtype=f64, device="cuda").unsqueeze(1).expand(-1, B, -1)
        out["rev"] = torch.func.vmap(vjp_fn)(eye)[0]                                             # [2n, B, 3]

    forward_mode()
    reverse_mode()
    err = float((out["fwd"].permute(1, 2, 0) - out["rev"].permute(1, 0, 2)).abs().max() / out["rev"].abs().max())
    return {"forward_mode_3_tangents": forward_mode, "reverse_mode_2n_cotangents": reverse_mode}, err


def report(scene, pairing, res, extra, args):
    out = {"scene": scene, "pairing": pairing, "unit": "ms", "card": card(), "rounds": args.rounds}
    out.update(extra)
    for k, v in res.items():
        out[k] = {"median": statistics.median(v), "min": min(v), "max": max(v)}
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=30)
    args = ap.parse_args()
    _lib.require_cuda()
    w = pile_world(args.batch, 24, 6, 2000)
    w.step()
    w.step()
    torch.cuda.synchronize()
    for R in (3, w.n):
        legs, held = kernel_legs(w, R)
        for fn in legs.values():
            fn()                                                   # warm-up
        torch.cuda.synchronize()
        res = {k: [] for k in legs}
        for _ in range(args.rounds):
            for k, fn in legs.items():
                res[k].append(timed(fn))
        report("%d piles of 24 balls" % args.batch, "(a) engine kernels, R = %d" % R, res,
               {"B": w.B, "n": w.n, "R": R, "mean_contacts_per_world": float(w.counts.float().mean())}, args)
    del w
    torch.cuda.empty_cache()
    for tag, (B, nb, cols, seed) in (("(b)", (args.batch, 24, 6, 2000)), ("(c)", (1, 60, 12, 4))):
        legs, err = rollout_legs(B, nb, cols, seed, args.steps)
        res = {k: [] for k in legs}
        for _ in range(args.rounds):
            for k, fn in legs.items():
                res[k].append(timed(fn))
        mem = {k + "_peak_MiB": peak(fn) for k, fn in legs.items()}
        scene = "%d piles of %d balls" % (B, nb) if B > 1 else "one %d-ball pile (banded kernel)" % nb
        report(scene, "%s d(state after %d steps)/d(friction, mass, velocity) per scene" % (tag, args.steps), res,
               dict(mem, B=B, n=3 * (nb + 1), steps=args.steps, forward_vs_reverse_rel_err=err), args)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
