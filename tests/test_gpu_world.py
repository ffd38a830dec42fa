"""GPU: `BatchedWorld` (B scenes in lock-step, fused engine kernels) reproduces the trajectories of B independent
unmodified reference `World`s (tests/golden/bworld_balls.npz, recorded by tests/golden/make_batched_world_golden.py):
six balls dropped onto a huge pinned ball, with and without post-stabilisation, 40 steps each, every scene with its
own contact set, contact count (0..3) and dt-halving history."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bworld_balls.npz")


@pytest.mark.parametrize("post_stab", [False, True])
def test_batched_world_reproduces_reference_worlds(post_stab):
    from lcp_physics_b200.world import BatchedWorld
    z = np.load(GOLDEN)
    t = lambda k: torch.from_numpy(z[k])
    world = BatchedWorld(t("pos"), t("rad"), vel=t("vel"), mass=t("mass"), restitution=t("rest"), fric_coeff=t("fric"),
                         gravity=100.0, static=[0], dt=1.0 / 30, post_stab=post_stab)
    tag = "ps" if post_stab else "nops"
    P, V, NC = t(tag + "_p"), t(tag + "_v"), t(tag + "_nc")
    worst_p, worst_v = 0.0, 0.0
    for k in range(P.shape[0]):
        world.step()
        assert torch.equal(world.counts.cpu().long(), NC[k].long()), (k, world.counts.tolist(), NC[k].tolist())
        worst_p = max(worst_p, float((world.p.cpu() - P[k]).abs().max()))
        worst_v = max(worst_v, float((world.v.cpu().reshape(P.shape[1], -1, 3) - V[k]).abs().max()))
    assert torch.allclose(world.t.cpu(), t(tag + "_t"), rtol=0, atol=1e-12)     # same dt-halving history
    assert worst_p < 1e-6 and worst_v < 1e-5, (worst_p, worst_v)                # positions O(300), velocities O(100)


def test_batched_world_is_differentiable():
    """Gradient of a final position w.r.t. an initial velocity flows through 12 steps (LCP backward on the GPU)."""
    from lcp_physics_b200.world import BatchedWorld
    z = np.load(GOLDEN)
    t = lambda k: torch.from_numpy(z[k])
    vel = t("vel").cuda().requires_grad_(True)
    world = BatchedWorld(t("pos"), t("rad"), vel=vel, mass=t("mass"), restitution=t("rest"), fric_coeff=t("fric"),
                         gravity=100.0, static=[0], dt=1.0 / 30)
    for _ in range(20):
        world.step()
    world.p[:, 1:, 1:].sum().backward()
    assert vel.grad is not None and torch.isfinite(vel.grad).all() and float(vel.grad.abs().max()) > 0


@pytest.mark.parametrize("nballs,cols,dtype", [(24, 6, torch.float64), (24, 6, torch.float32), (300, 20, torch.float64)])
def test_find_contacts_kernel_matches_torch_pair_scan(nballs, cols, dtype):
    """lcpb200_contacts' circle walk (pair test + ordered compaction, csrc/lcp_contacts.cuh) against the independent
    torch implementation (all-pairs tensors + stable sort): identical counts and identical ordered pair lists, on
    loose drops (0..few contacts per scene) and on a dense pile (~850 contacts)."""
    from lcp_physics_b200.scenes import make_ball_drop, make_ball_pile
    from lcp_physics_b200.world import BatchedWorld
    B = 9
    ic = make_ball_pile(B, nballs=nballs, cols=cols, seed=5, gap=0.05) if nballs > 100 else make_ball_drop(B, nballs=nballs, cols=cols, seed=5)
    if dtype == torch.float32:
        ic = {k: v.float() for k, v in ic.items()}
    w = BatchedWorld(ic["pos"], ic["rad"], vel=ic["vel"], mass=ic["mass"], restitution=ic["rest"], fric_coeff=ic["fric"],
                     gravity=100.0, static=[0], contact_capacity=4 * nballs)
    for step in range(6):
        counts, b1, b2 = w.find_contacts_torch()
        assert torch.equal(counts, w.counts), (step, counts.tolist(), w.counts.tolist())
        valid = torch.arange(w.cap, device=w.device).unsqueeze(0) < counts.unsqueeze(1)
        assert torch.equal(b1[valid], w.c_b1[valid]) and torch.equal(b2[valid], w.c_b2[valid])
        if nballs > 100:
            assert int(counts.min()) > 2 * nballs
        w.step()


def test_find_contacts_reports_overflow():
    from lcp_physics_b200.scenes import make_ball_pile
    from lcp_physics_b200.world import BatchedWorld
    ic = make_ball_pile(2, nballs=40, cols=8, seed=1, gap=0.05)
    with pytest.raises(RuntimeError, match="capacity"):
        BatchedWorld(ic["pos"], ic["rad"], gravity=100.0, static=[0], contact_capacity=16)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_fused_contact_geometry_matches_torch_geometry(dtype):
    """lcpb200_contacts' geometry (used when nothing needs autograd) against the differentiable torch geometry of the
    same selected pairs: normal, p1, p2, penetration, mu, restitution."""
    from lcp_physics_b200.scenes import make_ball_pile
    from lcp_physics_b200.world import BatchedWorld
    ic = make_ball_pile(7, nballs=40, cols=8, seed=9, gap=0.05)
    if dtype == torch.float32:
        ic = {k: v.float() for k, v in ic.items()}
    mk = lambda: BatchedWorld(ic["pos"], ic["rad"], vel=ic["vel"], mass=ic["mass"], restitution=ic["rest"],
                              fric_coeff=ic["fric"], gravity=100.0, static=[0], contact_capacity=160)
    a, b = mk(), mk()
    b.p.requires_grad_(True)                     # forces the torch (autograd) path
    b.find_contacts()
    assert b.c_normal.requires_grad and not a.c_normal.requires_grad
    assert torch.equal(a.counts, b.counts) and torch.equal(a.c_b1, b.c_b1) and torch.equal(a.c_b2, b.c_b2)
    tol = 1e-13 if dtype == torch.float64 else 1e-5
    valid = torch.arange(a.cap, device=a.device).unsqueeze(0) < a.counts.unsqueeze(1)
    for name in ("c_normal", "c_p1", "c_p2", "c_pen", "c_mu", "c_rest"):
        x, y = getattr(a, name), getattr(b, name).detach()
        assert torch.allclose(x[valid], y[valid], rtol=tol, atol=tol * 20), name
    assert bool((a.c_pen[~valid] < -1e29).all())
