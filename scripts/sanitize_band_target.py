"""Tiny banded-kernel calls for compute-sanitizer (memcheck / racecheck / synccheck): forward + backward of the
large-scene kernels forced onto small scenes (with equality rows and per-scene counts), one step of a 60-ball
world (n = 183: natively banded, includes lcpb200_contacts)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ["LCPB200_FORCE_BANDED"] = "1"
import torch
from lcp_physics_b200.engines import engine_solve
from lcp_physics_b200.scenes import make_contact_soa, make_ball_pile
from lcp_physics_b200.world import BatchedWorld

which = sys.argv[1] if len(sys.argv) > 1 else "small"
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 2
if which == "small":
    B, nb, nc, e = 3, 12, 20, 3
    soa = make_contact_soa(B, nb, nc, seed=2)
    fext = torch.zeros(B, 3 * nb, dtype=torch.float64)
    fext[:, 2::3] = 10.0 * soa["mass"]
    names = ["mass", "inertia", "v", "fext", "normal", "p1", "p2", "mu", "restitution"]
    for mode in (0, 1):
        lv = [(fext if k == "fext" else soa[k]).cuda().requires_grad_(True) for k in names]
        A = torch.zeros(B, e, 3 * nb, dtype=torch.float64)
        A[:, torch.arange(e), torch.arange(e)] = 1
        A = A.cuda().requires_grad_(True)
        b = torch.zeros(B, e, dtype=torch.float64).cuda().requires_grad_(True)
        b1 = soa["body1"].unsqueeze(0).expand(B, -1).contiguous().cuda()
        b2 = soa["body2"].unsqueeze(0).expand(B, -1).contiguous().cuda()
        counts = torch.tensor([nc, nc - 5, 0], dtype=torch.int32).cuda()
        z, st = engine_solve(*lv, b1, b2, 1.0 / 30, A=A, b=b, mode=mode, max_iter=iters, counts=counts)
        z.sum().backward()
        torch.cuda.synchronize()
        print("done small mode", mode, st.tolist())
else:
    ic = make_ball_pile(1, nballs=60, cols=10, seed=3, gap=0.05)
    w = BatchedWorld(ic["pos"], ic["rad"], vel=ic["vel"], mass=ic["mass"], restitution=ic["rest"], fric_coeff=ic["fric"],
                     gravity=100.0, static=[0], contact_capacity=200, max_iter=iters)
    w.step()
    torch.cuda.synchronize()
    print("done world", w.counts.tolist())
