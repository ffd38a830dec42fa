"""GPU: cost of the exact adjoint against the reference's (bug-compatible) adjoint in the engine backward.

Both flags factor the KKT matrix once per backward (K or K^T), so the expectation is equal cost. The script times
`engine_solve`'s backward (lcpb200_engine_backward) with CUDA events, the two flags alternated in one process, on
  * the `bench.py --config world` shape: 1024 piles of 24 balls on a pinned floor ball (condensed kernel);
  * one BASELINE config-4 pile of 512 balls (banded kernel).
The forward runs once per flag; its autograd graph is kept and the backward replayed. Prints one JSON line with the
GPU name and power limit next to the medians.

    python scripts/exact_adjoint_cost.py [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lcp_physics_b200.engines import engine_solve  # noqa: E402
from lcp_physics_b200.scenes import make_ball_pile  # noqa: E402
from lcp_physics_b200.world import BatchedWorld  # noqa: E402


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:
        return None


def graphs(ic, cap):
    """One forward per flag from the initial contact list of a BatchedWorld; returns {exact: (zhat, dl/dzhat)}."""
    w = BatchedWorld(ic["pos"], ic["rad"], vel=ic["vel"], mass=ic["mass"], restitution=ic["rest"],
                     fric_coeff=ic["fric"], gravity=100.0, static=[0], dt=1.0 / 30, contact_capacity=cap)
    b = torch.zeros(w.B, w.ne, dtype=w.dtype, device=w.device)
    g = torch.randn(w.B, w.n, dtype=w.dtype, generator=torch.Generator().manual_seed(0)).to(w.device)
    out = {}
    for exact in (False, True):
        leaves = [t.detach().clone().requires_grad_(True)
                  for t in (w.mass, w.inertia, w.v, w.fext, w.c_normal, w.c_p1, w.c_p2, w.c_mu, w.c_rest)]
        z, st = engine_solve(*leaves, w.c_b1, w.c_b2, w.dt, A=w.A, b=b, mode=0, max_iter=w.max_iter,
                             exact_adjoint=exact, counts=w.counts)
        assert bool((st >= 0).all()), st
        out[exact] = (z, g)
    return out, w


def time_backward(gr, reps):
    ev = lambda: torch.cuda.Event(enable_timing=True)
    for exact in (False, True):                               # warm-up: handles, workspaces
        gr[exact][0].backward(gr[exact][1], retain_graph=True)
    ms = {False: [], True: []}
    for r in range(reps):
        for exact in ((False, True) if r % 2 == 0 else (True, False)):
            z, g = gr[exact]
            e0, e1 = ev(), ev()
            torch.cuda.synchronize()
            e0.record()
            z.backward(g, retain_graph=True)
            e1.record()
            torch.cuda.synchronize()
            ms[exact].append(e0.elapsed_time(e1))
    med = lambda v: sorted(v)[len(v) // 2]
    return {"bug_compatible_ms": med(ms[False]), "exact_ms": med(ms[True]),
            "exact_over_bug_compatible": med(ms[True]) / med(ms[False]), "reps": reps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    res = {"gpu": torch.cuda.get_device_name(), "power_limit_w": power_limit_w(),
           "timed": "engine_solve backward (lcpb200_engine_backward + autograd glue), CUDA events, flags alternated, "
                    "median over reps"}
    gr, w = graphs(make_ball_pile(1024, nballs=24, cols=6, seed=2000, gap=0.05), None)
    res["world_1024x24_condensed"] = dict(time_backward(gr, args.reps), large=w.large,
                                          mean_contacts=float(w.counts.float().mean()))
    del gr, w
    gr, w = graphs(make_ball_pile(1, nballs=512, cols=32, seed=3000, gap=0.05), 4 * 512)
    res["cfg4_512_banded"] = dict(time_backward(gr, args.reps), large=w.large, contacts=int(w.counts[0]))
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
