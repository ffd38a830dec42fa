"""Cost of Jacobians through LCPFunction (the dense path): one batched call against one call per right-hand side.

  (1) one lcpb200_backward_batched call with R = n cotangents against R lcpb200_backward calls, on the same saved
      solve (outputs dp and dh, preallocated for every leg);
  (2) one lcpb200_jvp_batched call with R tangents (of p, h and b) against R single-tangent calls, R = 3 and R = n;
  (3) jacrev of zhat w.r.t. (p, h) -- n one-hot cotangents placed in every scene at once, one torch.func.vmap of the
      VJP -- against n torch.autograd.grad calls.
Shapes: "cfg3" (bench.py config 3's n = 96, m = 256, fp32, condensed kernel; 1024 scenes), "contacts_f64" (n = 48,
m = 128 contact scenes in fp64: dual form first; 256 scenes), "dense_f64" (scenes.make_dense_random, n = 32, m = 48,
fp64: dual form only; 256 scenes). Legs of a pairing alternate inside every round (CUDA events). One JSON line per
pairing: median and spread (min, max) of every leg, the card and its power limit. With --out DIR the lines are also
written to DIR/lcp_jacobian_bench.jsonl; nothing else is written.

    python scripts/lcp_jacobian_bench.py [--rounds 5] [--shapes cfg3,contacts_f64,dense_f64] [--out DIR]
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lcp_physics_b200 import LCPFunction, _lib  # noqa: E402
from lcp_physics_b200.scenes import make_dense_random, make_scenes  # noqa: E402
from scripts.obstacle_bench import card  # noqa: E402

SHAPES = {
    "cfg3": lambda: make_scenes(1024, 32, 64, fd=2, dtype=torch.float32, seed=0),
    "contacts_f64": lambda: make_scenes(256, 16, 32, fd=2, dtype=torch.float64, seed=0),
    "dense_f64": lambda: make_dense_random(256, 32, 48, dtype=torch.float64, seed=0),
}


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def pairing(legs, rounds):
    for fn in legs.values():
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in legs}
    for _ in range(rounds):
        for k, fn in legs.items():
            times[k].append(timed(fn))
    return {k: {"median": statistics.median(v), "min": min(v), "max": max(v)} for k, v in times.items()}


def emit(line, out):
    s = json.dumps(line)
    print(s, flush=True)
    if out:
        with open(os.path.join(out, "lcp_jacobian_bench.jsonl"), "a") as f:
            f.write(s + "\n")


def run_shape(name, rounds, out):
    lib = _lib.load()
    ins = [t.cuda().contiguous() for t in SHAPES[name]()]
    Q, p, G, h, A, b, F = ins
    dtype = Q.dtype
    B, m, n = G.shape
    hd = _lib.get_handle(dtype, n, m, 0, torch.cuda.current_device(), torch.cuda.current_stream().cuda_stream)
    mk = lambda *s, d=dtype: torch.empty(*s, dtype=d, device="cuda")
    zhat, lam, slack = mk(B, n), mk(B, m), mk(B, m)
    status, iters, resid = mk(B, d=torch.int32), mk(B, d=torch.int32), mk(B)
    ptr = _lib.ptr
    _lib.check(lib.lcpb200_forward(hd.raw, B, *[ptr(t) for t in (Q, p, G, h, None, None, F)], 1e-12, 3, 10,
                                   *[ptr(t) for t in (zhat, None, lam, slack, status, iters, resid, None)], None))
    torch.cuda.synchronize()
    base = dict(shape=name, B=B, n=n, m=m, dtype=str(dtype).split(".")[-1], card=card(), rounds=rounds, unit="ms",
                describe=hd.describe())
    common = [ptr(t) for t in (Q, G, None, F, zhat, None, lam, slack)]

    # (1) R = n cotangents: one batched call against R single calls
    R = n
    g = torch.randn(R, B, n, dtype=dtype, device="cuda")
    dp, dh = mk(R, B, n), mk(R, B, m)

    def bwd_batched():
        _lib.check(lib.lcpb200_backward_batched(hd.raw, R, B, *common, ptr(g), None, ptr(dp), None, ptr(dh), None, None,
                                                None, None, 0, None))

    def bwd_single():
        for r in range(R):
            _lib.check(lib.lcpb200_backward(hd.raw, B, *common, ptr(g[r]), None, ptr(dp[r]), None, ptr(dh[r]), None,
                                            None, None, None, 0, None))
    emit(dict(base, pairing="vjp R=n: one batched call vs R single calls", R=R,
              **pairing({"batched": bwd_batched, "single": bwd_single}, rounds)), out)

    # (2) R tangents of p and h: one batched call against R single-tangent calls
    for R in (3, n):
        tp, th = torch.randn(R, B, n, dtype=dtype, device="cuda"), torch.randn(R, B, m, dtype=dtype, device="cuda")
        dz = mk(R, B, n)

        def jvp_batched():
            _lib.check(lib.lcpb200_jvp_batched(hd.raw, R, B, *common, None, ptr(tp), None, ptr(th), None, None, None,
                                               ptr(dz), None, 0, None))

        def jvp_single():
            for r in range(R):
                _lib.check(lib.lcpb200_jvp_batched(hd.raw, 1, B, *common, None, ptr(tp[r]), None, ptr(th[r]), None,
                                                   None, None, ptr(dz[r]), None, 0, None))
        emit(dict(base, pairing="jvp R=%d: one batched call vs R single-tangent calls" % R, R=R,
                  **pairing({"batched": jvp_batched, "single": jvp_single}, rounds)), out)

    # (3) jacrev w.r.t. (p, h): vmap of one VJP over n one-hot cotangents against n autograd.grad calls
    fn = LCPFunction(max_iter=10)
    pl, hl = p.clone().requires_grad_(True), h.clone().requires_grad_(True)
    eye = torch.eye(n, dtype=dtype, device="cuda")[:, None, :].expand(n, B, n).contiguous()

    def jac_vmap():
        _, vjp_fn = torch.func.vjp(lambda p_, h_: fn(Q, p_, G, h_, A, b, F), p, h)
        torch.func.vmap(vjp_fn)(eye)

    def jac_loop():
        z = fn(Q, pl, G, hl, A, b, F)
        for r in range(n):
            torch.autograd.grad(z, (pl, hl), eye[r], retain_graph=r + 1 < n)
    emit(dict(base, pairing="jacrev (p, h): vmap of one VJP vs n autograd.grad calls (each leg includes its forward)",
              R=n, **pairing({"vmap": jac_vmap, "loop": jac_loop}, rounds)), out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    _lib.require_cuda()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
    for name in args.shapes.split(","):
        run_shape(name, args.rounds, args.out)


if __name__ == "__main__":
    main()
