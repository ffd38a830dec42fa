"""Development check of the condensed-KKT kernels on a GPU box: parity vs the oracle + timing."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from lcp_physics_b200 import solve_forward, solve_backward, _lib
from lcp_physics_b200.scenes import make_scenes
from oracle import pdipm_oracle as po


def rel(a, b):
    a = a.double().reshape(a.shape[0], -1); b = b.double().reshape(b.shape[0], -1)
    return (a - b).norm(dim=1) / b.norm(dim=1).clamp_min(1e-300)


def check(name, nb, nc, fd, e, dtype, B=16, mi=10):
    inp64 = make_scenes(B, nb, nc, fd=fd, e=e, dtype=torch.float64, seed=101)
    inp = tuple(t.to(dtype) for t in inp64)
    ref = po.lcp_forward(*inp64, max_iter=mi, coupled=False)
    t0 = time.time()
    out = solve_forward(*[t.cuda() for t in inp], max_iter=mi)
    torch.cuda.synchronize()
    zhat, nu, lam, slack, status, iters, resid = out
    err = rel(zhat.cpu(), ref.zhat)
    print("%-22s %s: zhat err med %.1e max %.1e | status %s iters %.1f (ref %.1f) | %s" % (
        name, str(dtype)[-7:], err.median(), err.max(), sorted(set(status.cpu().tolist())), iters.float().mean(),
        ref.info["iters"].float().mean(), _lib.get_handle(dtype, 3 * nb, nc * (2 + fd), e, 0).describe()[:140]), flush=True)
    if dtype == torch.float32:
        g = torch.randn(B, 3 * nb, generator=torch.Generator().manual_seed(1))
        Q, p, G, h, A, b, F = [t.cuda() for t in inp]
        gr = solve_backward(Q, G, A if e else None, F, zhat, nu, lam, slack, g.cuda())
        st64 = [None if t is None else t.cpu().double() for t in (zhat, nu, lam, slack)]
        rg = po.lcp_backward_from_saved(inp64, st64[0], st64[1], st64[2], st64[3], g.double())
        for nm, a, b_ in zip("dQ dp dG dh dA db dF".split(), gr, rg):
            if a is None: continue
            er = rel(a.cpu(), b_)
            print("      bwd %s vs fp64 oracle (same state): med %.1e max %.1e" % (nm, er.median(), er.max()))


if __name__ == "__main__":
    torch.cuda.set_device(0)
    check("small e0", 4, 4, 2, 0, torch.float64)
    check("small e3", 4, 4, 2, 3, torch.float64)
    check("odd", 5, 7, 2, 3, torch.float64)
    check("cfg2 shape", 16, 32, 3, 0, torch.float64)
    check("cfg3 shape f64", 32, 64, 2, 0, torch.float64)
    check("cfg3 e3 f64", 32, 64, 2, 3, torch.float64)
    check("cfg3 shape f32", 32, 64, 2, 0, torch.float32, B=32)
    check("cfg3 e3 f32", 32, 64, 2, 3, torch.float32)
    check("cfg2 shape f32", 16, 32, 3, 0, torch.float32)
    # timing at the BASELINE size
    B = 4096
    inp = [t.cuda() for t in make_scenes(B, 32, 64, fd=2, e=0, dtype=torch.float32, seed=7)]
    hd = _lib.get_handle(torch.float32, 96, 256, 0, 0)
    for rep in range(4):
        if rep == 3:
            hd.profile(True)
        torch.cuda.synchronize(); t0 = time.time()
        out = solve_forward(*inp, max_iter=10)
        torch.cuda.synchronize(); t1 = time.time()
        g = torch.randn(B, 96, device="cuda")
        gr = solve_backward(inp[0], inp[2], None, inp[6], out[0], None, out[2], out[3], g)
        torch.cuda.synchronize(); t2 = time.time()
        print("cfg3 B=4096: forward %.2f ms  backward %.2f ms  status %s iters %.2f" % (
            (t1 - t0) * 1e3, (t2 - t1) * 1e3, sorted(set(out[4].cpu().tolist())), out[5].float().mean()), flush=True)
    pr = hd.profile(False)
    tot = sum(v for k, v in pr.items() if k.startswith("c_"))
    print("condensed phases (share of counted cycles, cycles per scene):")
    for k, v in pr.items():
        if k.startswith("c_") and v:
            print("   %-18s %5.1f %%  %9.0f" % (k, 100.0 * v / tot, v / B))
    print("executed per scene: %.2f factorisations, %.2f solves" % (pr["factorisations"] / B, pr["solves"] / B))
    for Bs in (132, 264):
        sub = [t[:Bs].contiguous() for t in inp]
        solve_forward(*sub, max_iter=10)
        hd.profile(True)
        torch.cuda.synchronize(); t0 = time.time()
        solve_forward(*sub, max_iter=10)
        torch.cuda.synchronize(); t1 = time.time()
        pr = hd.profile(False)
        print("forward only, B=%d (%.2f ms): cycles per scene:" % (Bs, (t1 - t0) * 1e3),
              " ".join("%s=%.0f" % (k[2:], v / Bs) for k, v in pr.items() if k.startswith("c_") and v),
              "| per scene: %.2f factorisations, %.2f solves" % (pr["factorisations"] / Bs, pr["solves"] / Bs))
    B = 1024
    inp = [t.cuda() for t in make_scenes(B, 16, 32, fd=3, e=0, dtype=torch.float64, seed=7)]
    for rep in range(3):
        torch.cuda.synchronize(); t0 = time.time()
        out = solve_forward(*inp, max_iter=10)
        torch.cuda.synchronize(); t1 = time.time()
        print("cfg2 B=1024 fp64: forward %.2f ms status %s" % ((t1 - t0) * 1e3, sorted(set(out[4].cpu().tolist()))), flush=True)
