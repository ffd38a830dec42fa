"""Signed distances and images of `BatchedWorld` scenes (lcpb200_signed_distance, `signed_distance`, `render`), timed on
the GPU.

* (a) 1024 piles of 24 balls in a bin of 3 obstacles, one window over the bin for the whole batch:
    render_hard     `render(64, 64)` with nothing differentiated (sigma = 0);
    render_soft_bwd `render(64, 64, sigma=2)` with the state requiring grad, then a backward pass of the image's sum;
    sdf_256         `signed_distance` of 256 points shared by the batch, nothing differentiated;
    sdf_ref_256     the dense brute force of tests/sdf_ref.py on the same points, on the same GPU;
* (b) one 512-ball pile (BASELINE config 4) at `render(512, 512)`: hard, and soft with a backward pass;
* (c) one hard `render(64, 64)` call against one `step()` of the worlds in (a).
Legs of a pairing alternate inside every round; prints one JSON line per pairing with the median and the spread
(min, max) of every leg, and the card and its power limit read in the same run.

    python scripts/sdf_bench.py [--rounds 5] [--calls 20] [--warmup 3] [--batch 1024]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lcp_physics_b200.scenes import make_ball_pile  # noqa: E402
from lcp_physics_b200.world import BatchedWorld  # noqa: E402
from scripts.hetero_bench import G, balls, bin_obstacles  # noqa: E402
from scripts.raycast_bench import pairing  # noqa: E402
from tests.sdf_ref import sdf_ref  # noqa: E402


def window(w):
    """the bounding box of every body of every scene, 10 units of margin"""
    pts = [w.p[:, :w.nb, 1:] - w.rad.unsqueeze(2), w.p[:, :w.nb, 1:] + w.rad.unsqueeze(2)]
    if w.no:
        pts.append(w.ov.reshape(w.B, -1, 2))
    pts = torch.cat(pts, 1).detach().reshape(-1, 2)
    return pts.min(0).values - 10.0, pts.max(0).values + 10.0


def render_legs(w, H, W, lo, hi, sigma=2.0):
    p_leaf = w.p.detach().clone().requires_grad_()

    def hard():
        with torch.no_grad():
            w.render(H, W, lo, hi)

    def soft_bwd():
        p0 = w.p
        w.p = p_leaf
        try:
            img, _, _ = w.render(H, W, lo, hi, sigma=sigma)
            img.sum().backward()
        finally:
            w.p = p0
    return {"render_hard": hard, "render_soft_bwd": soft_bwd}


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
    lo, hi = window(w)
    md = float((hi - lo).norm())
    # (a) the kernel path, the graph path and the brute force agree before they are timed
    g = torch.Generator(device=w.device).manual_seed(0)
    x = lo + (hi - lo) * torch.rand(256, 2, generator=g, dtype=w.dtype, device=w.device)
    with torch.no_grad():
        sk, bk, _ = w.signed_distance(x, md)
        rs, rb, _, _, margin = sdf_ref(w.p[:, :w.nb, 1:], w.rad, None, w.ov, x.expand(B, -1, -1), md, chunk=64)
    ok = margin > 1e-9
    assert torch.equal(bk[ok], rb[ok]) and float((sk - rs).abs().max()) < 1e-9
    xg = x.clone().requires_grad_()
    sg, bg, _ = w.signed_distance(xg, md)
    assert torch.equal(bk, bg) and float((sk - sg.detach()).abs().max()) < 1e-9
    with torch.no_grad():
        img, body, _ = w.render(64, 64, lo, hi)

    def sdf_256():
        with torch.no_grad():
            w.signed_distance(x, md)

    def ref_256():
        with torch.no_grad():
            sdf_ref(w.p[:, :w.nb, 1:], w.rad, None, w.ov, x.expand(B, -1, -1), md, chunk=64)
    legs = render_legs(w, 64, 64, lo, hi)
    legs.update({"sdf_256": sdf_256, "sdf_ref_256": ref_256})
    pairing("(a) %d piles of 24 balls in a 3-obstacle bin: render(64, 64), 256 shared points" % B, legs, args,
            {"B": B, "pixels": B * 64 * 64, "lit_fraction": float(img.mean()), "decided_fraction": float(ok.float().mean()),
             "bodies_seen": int(body.unique().numel())})
    # (b) one 512-ball pile at 512 x 512
    ic1 = make_ball_pile(1, nballs=512, cols=32, seed=0)
    w1 = BatchedWorld(ic1["pos"], ic1["rad"], vel=ic1["vel"], mass=ic1["mass"], restitution=ic1["rest"],
                      fric_coeff=ic1["fric"], gravity=G, static=[0], dt=1.0 / 30)
    lo1, hi1 = window(w1)
    pairing("(b) one 512-ball pile, render(512, 512)", render_legs(w1, 512, 512, lo1, hi1), args,
            {"B": 1, "pixels": 512 * 512})
    # (c) one hard render against one step of the worlds in (a)
    wc = BatchedWorld(gravity=G, dt=1.0 / 30, obstacles=bin_obstacles(ic), **balls(ic))

    def render():
        with torch.no_grad():
            wc.render(64, 64, lo, hi)

    def step():
        with torch.no_grad():
            wc.step()
    out = pairing("(c) one render(64, 64) vs one step(), %d piles of 24 balls" % B, {"render": render, "step": step},
                  args, {"B": B})
    print(json.dumps({"render_over_step": out["render"]["ms_median"] / out["step"]["ms_median"]}), flush=True)


if __name__ == "__main__":
    main()
