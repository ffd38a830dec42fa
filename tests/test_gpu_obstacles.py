"""GPU: static convex polygon obstacles in `BatchedWorld` (one-body contacts, body2 >= nb).

* lcpb200_contacts' pair lists / counts equal `find_contacts_torch`'s bitwise (several 1024-pair chunks,
  fp64 / fp32), its geometry equals the differentiable torch geometry (outside and centre-inside cases) and the
  contact list the unmodified reference recorded (tests/golden/bworld_obstacles.npz);
* engine_solve with one-body contacts equals the reference's pinned formulation (the obstacle an extra body with
  TotalConstraint rows), both modes, both adjoints, condensed and banded kernels;
* the 16 recorded engine calls of tests/golden/world_large.npz (60 circles on a pinned `Rect` floor) are reproduced
  with the floor as a static obstacle (its dofs and Je dropped, floor contacts turned into one-body contacts);
* `BatchedWorld(obstacles=...)` reproduces the reference's trajectories; a 150-ball pile in a bin of 6 obstacles
  (banded kernel) agrees with oracle/obstacle_oracle.py; rollout gradients w.r.t. a ramp's angle and friction agree
  with central differences.
"""
import math
import os

import numpy as np
import pytest
import torch

from tests.helpers import load_world_records

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bworld_obstacles.npz")


@pytest.fixture
def forced_banded():
    from lcp_physics_b200 import _lib

    def set_(on):
        if on:
            os.environ["LCPB200_FORCE_BANDED"] = "1"
        else:
            os.environ.pop("LCPB200_FORCE_BANDED", None)
        _lib.clear_handles()
    yield set_
    set_(False)


def golden_world(z, post_stab=False, **kw):
    from lcp_physics_b200.world import BatchedWorld
    t = lambda k: torch.from_numpy(z[k])
    return BatchedWorld(t("pos"), t("rad"), vel=t("vel"), mass=t("mass"), restitution=t("rest"), fric_coeff=t("fric"),
                        gravity=100.0, dt=1.0 / 30, post_stab=post_stab, obstacles=t("obst_verts"),
                        obstacle_fric=t("obst_fric"), obstacle_rest=t("obst_rest"), **kw)


def bin_scene(B, nballs, cols, rad=10.0, seed=0, dtype=torch.float64):
    """A square-stacked pile of nballs circles resting on a floor between two walls (gaps 0.02..0.06 < eps), and
    three more obstacles above the pile (a triangle, a pentagon, a tilted rect): 6 static obstacles."""
    from lcp_physics_b200.world import rect_vertices
    g = torch.Generator().manual_seed(seed)
    rows = (nballs + cols - 1) // cols
    floor_y, x0 = 500.0, 100.0
    pos = torch.zeros(B, nballs, 2, dtype=torch.float64)
    for k in range(nballs):
        r_, c_ = divmod(k, cols)
        pos[:, k, 0] = x0 + rad + 2 * rad * c_ + 0.05 * c_
        pos[:, k, 1] = floor_y - rad - 0.04 - (2 * rad + 0.05) * r_
    pos[:, :, 0] += 0.01 * torch.rand(B, nballs, generator=g, dtype=torch.float64)
    width = 2 * rad * cols + 0.05 * (cols - 1)
    top = floor_y - (2 * rad + 0.05) * rows
    tri = torch.tensor([[0.0, 0.0], [40.0, 0.0], [20.0, -30.0]], dtype=torch.float64) + torch.tensor([x0, top - 80.0])
    ang = torch.arange(5, dtype=torch.float64) * (2 * math.pi / 5)
    pent = torch.stack([torch.cos(ang), torch.sin(ang)], 1) * 20.0 + torch.tensor([x0 + width / 2, top - 90.0])
    quads = [rect_vertices([x0 + width / 2, floor_y + 10.0], [width + 100.0, 20.0]),                    # floor
             rect_vertices([x0 - 10.0 - 0.03, floor_y - 141.0], [20.0, 280.0]),                          # walls
             rect_vertices([x0 + width + 10.0 + 0.03, floor_y - 141.0], [20.0, 280.0]),
             rect_vertices([x0 + width - 40.0, top - 70.0], [50.0, 8.0], 0.4)]
    obst = [_pad(o, 5) for o in (quads[0], quads[1], quads[2], tri, pent, quads[3])]
    return dict(pos=pos.to(dtype), rad=torch.full((B, nballs), rad, dtype=dtype), obst=torch.stack(obst))


# ---------------------------------------------------------------------------------------------------- contact lists
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_world_contacts_kernel_matches_torch_pair_scan(dtype):
    """fp64: 150 circles + 6 obstacles, 11 175 + 900 pairs per scene, 12 chunks of 1024 pairs (banded kernel);
    fp32 (condensed kernels: 3 nb <= 128): 42 circles + 6 obstacles, 861 + 252 pairs, 2 chunks."""
    from lcp_physics_b200.world import BatchedWorld
    big = dtype == torch.float64
    sc = bin_scene(3, 150, 15, dtype=dtype) if big else bin_scene(3, 42, 14, dtype=dtype)
    for ob in (sc["obst"].to(dtype), sc["obst"][:3].to(dtype)):
        w = BatchedWorld(sc["pos"], sc["rad"], gravity=100.0, obstacles=ob, contact_capacity=800 if big else 160,
                         strict_no_penetration=False)
        assert int(w.pi.numel()) > (10 if big else 1) * 1024 or ob.shape[0] == 3
        for step in range(4):
            counts, b1, b2 = w.find_contacts_torch()
            assert torch.equal(counts, w.counts), (step, counts.tolist(), w.counts.tolist())
            valid = torch.arange(w.cap, device=w.device).unsqueeze(0) < counts.unsqueeze(1)
            assert torch.equal(b1[valid], w.c_b1[valid]) and torch.equal(b2[valid], w.c_b2[valid])
            w.step()


def test_world_contacts_reports_overflow():
    from lcp_physics_b200.world import BatchedWorld
    sc = bin_scene(2, 60, 12)
    with pytest.raises(RuntimeError, match="capacity"):
        BatchedWorld(sc["pos"], sc["rad"], gravity=100.0, obstacles=sc["obst"][:3], contact_capacity=16)


# ---------------------------------------------------------------------------------------------------- geometry
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_world_contact_geometry_kernel_matches_torch(dtype):
    """Shallow contacts and centre-inside (SAT) contacts: kernel path (no autograd) against the torch path."""
    from lcp_physics_b200.world import BatchedWorld, rect_vertices
    box = rect_vertices([0.0, 0.0], [100.0, 40.0], 0.2)
    tri = torch.tensor([[150.0, 0.0], [210.0, 10.0], [170.0, -50.0]], dtype=torch.float64)
    # a triangle padded to V = 4 by repeating a vertex (zero-length edge): skipped by both paths
    pad = torch.tensor([[0.0, 100.0], [40.0, 100.0], [20.0, 130.0], [20.0, 130.0]], dtype=torch.float64)
    obst = torch.stack([box, torch.stack([tri[0], tri[1], 0.5 * (tri[1] + tri[2]) + torch.tensor([0.5, 0.0]), tri[2]]),
                        pad])
    pos = torch.tensor([[[0.0, -29.0], [30.0, 5.0], [-45.0, 3.0], [180.0, -10.0], [215.0, 12.0], [260.0, 0.0],
                         [55.0, -30.0], [20.0, 112.0], [20.0, 139.5], [-9.0, 100.0]]], dtype=torch.float64)
    pos = pos.expand(2, -1, -1).clone()
    pos[1] += 0.7
    rad = torch.full((2, pos.shape[1]), 10.0, dtype=torch.float64)
    mk = lambda: BatchedWorld(pos.to(dtype), rad.to(dtype), gravity=100.0, obstacles=obst.to(dtype),
                              obstacle_fric=torch.tensor([0.3, 0.7, 0.5]), obstacle_rest=torch.tensor([0.1, 0.4, 0.2]),
                              strict_no_penetration=False, contact_capacity=40)
    a, b = mk(), mk()
    b.ov.requires_grad_(True)
    b.find_contacts()
    counts, b1, b2 = a.find_contacts_torch()
    assert torch.equal(counts, a.counts)
    assert int(((a.c_b2 == a.nb + 2) & (torch.arange(a.cap, device=a.device) < a.counts.unsqueeze(1))).sum()) >= 4
    for name in ("c_normal", "c_p1", "c_p2", "c_pen"):
        assert bool(torch.isfinite(getattr(b, name)).all()), name
    valid_b = torch.arange(b.cap, device=b.device).unsqueeze(0) < b.counts.unsqueeze(1)
    (b.c_pen[valid_b].sum() + b.c_normal[valid_b].sum()).backward()
    assert bool(torch.isfinite(b.ov.grad).all()) and float(b.ov.grad[:, 2].abs().sum()) > 0
    assert b.c_normal.requires_grad and not a.c_normal.requires_grad
    assert torch.equal(a.counts, b.counts) and torch.equal(a.c_b1, b.c_b1) and torch.equal(a.c_b2, b.c_b2)
    valid = torch.arange(a.cap, device=a.device).unsqueeze(0) < a.counts.unsqueeze(1)
    obs = valid & (a.c_b2 >= a.nb)
    assert int(obs.sum()) >= 4 and bool((a.c_pen[obs] > 10.0).any())             # centre-inside contacts present
    tol = 1e-12 if dtype == torch.float64 else 1e-6
    for name in ("c_normal", "c_p1", "c_p2", "c_pen", "c_mu", "c_rest"):
        x, y = getattr(a, name), getattr(b, name).detach()
        scale = max(1.0, float(x[valid].abs().max()))
        assert float((x[valid] - y[valid]).abs().max()) <= tol * scale, name
    assert bool((a.c_pen[~valid] < -1e29).all())


def test_world_contact_geometry_matches_reference_contact_list():
    z = np.load(GOLDEN)
    for grad in (False, True):
        w = golden_world(z)
        if grad:
            w.ov.requires_grad_(True)
            w.find_contacts()
        for s in range(z["pos"].shape[0]):
            n = int(z["first_n"][s])
            assert int(w.counts[s]) == n
            assert w.c_b1[s, :n].cpu().tolist() == z["first_b1"][s, :n].tolist()
            assert w.c_b2[s, :n].cpu().tolist() == z["first_b2"][s, :n].tolist()
            for name, key in (("c_normal", "normal"), ("c_p1", "p1"), ("c_p2", "p2"), ("c_pen", "pen")):
                x = getattr(w, name)[s, :n].detach().cpu().numpy()
                assert np.abs(x - z["first_" + key][s, :n]).max() < 1e-9, (grad, name)


# ---------------------------------------------------------------------------------------------------- reduced vs pinned
def _pinned_inputs(w):
    """The same contacts in the reference's formulation: obstacle k becomes body nb + k (mass 1, Rect inertia),
    pinned by TotalConstraint rows."""
    from oracle.obstacle_oracle import hull_inertia
    B, nb, no = w.B, w.nb, w.no
    dev, dt_ = w.device, w.dtype
    mass = torch.cat([w.mass, torch.ones(B, no, dtype=dt_, device=dev)], 1)
    inert = torch.stack([hull_inertia((w.ov[0, k] - w.oref[0, k]).detach().cpu().double(), 1.0) for k in range(no)])
    inertia = torch.cat([w.inertia, inert.to(dev, dt_).unsqueeze(0).expand(B, -1)], 1)
    v = torch.cat([w.v, torch.zeros(B, 3 * no, dtype=dt_, device=dev)], 1)
    fext = torch.cat([w.fext, torch.zeros(B, 3 * no, dtype=dt_, device=dev)], 1)
    A = torch.zeros(B, 3 * no, 3 * (nb + no), dtype=dt_, device=dev)
    for r in range(3 * no):
        A[:, r, 3 * nb + r] = 1.0
    return mass, inertia, v, fext, A


@pytest.mark.parametrize("banded", [False, True])
@pytest.mark.parametrize("exact", [False, True])
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_one_body_contacts_equal_pinned_formulation(forced_banded, banded, exact, mode, dtype):
    """banded: the reduced formulation through the large-scene kernel. The pinned formulation always goes through the
    condensed kernel: its 4 pinned obstacles need 24 border rows, more than the banded kernel's 16."""
    from lcp_physics_b200.engines import engine_solve
    if banded and dtype == torch.float32:
        pytest.skip("the large-scene kernel is fp64 only")
    z = np.load(GOLDEN)
    w = golden_world(z)
    for _ in range(3):
        w.step()
    B, nb, n = w.B, w.nb, w.n
    cast = lambda t: t.to(dtype).detach()
    mass, inertia, v, fext, A = [cast(t) for t in _pinned_inputs(w)]
    geo = {k: cast(getattr(w, "c_" + k)).requires_grad_(True) for k in ("normal", "p1", "p2", "mu", "rest")}
    geo2 = {k: t.detach().clone().requires_grad_(True) for k, t in geo.items()}
    vr, vp = cast(w.v).requires_grad_(True), v.clone().requires_grad_(True)
    dt = 1.0 / 30 if mode == 0 else 0.0
    wgt = torch.linspace(-1.0, 1.0, n, dtype=dtype, device=w.device)
    forced_banded(banded)
    zr, sr = engine_solve(cast(w.mass), cast(w.inertia), vr, cast(w.fext), geo["normal"], geo["p1"], geo["p2"], geo["mu"],
                          geo["rest"], w.c_b1, w.c_b2, dt, mode=mode, exact_adjoint=exact, counts=w.counts)
    (zr * wgt).sum().backward()
    forced_banded(False)
    zp, sp = engine_solve(mass, inertia, vp, fext, geo2["normal"], geo2["p1"], geo2["p2"], geo2["mu"], geo2["rest"],
                          w.c_b1, w.c_b2, dt, A=A, b=torch.zeros(B, A.shape[1], dtype=dtype, device=w.device), mode=mode,
                          exact_adjoint=exact, counts=w.counts)
    assert bool((sr >= 0).all()) and bool((sp >= 0).all()), (sr.tolist(), sp.tolist())
    rel = float((zr - zp[:, :n]).norm() / zp[:, :n].norm().clamp_min(1e-30))
    print("zhat relative difference (dtype %s, mode %d, banded %s): %.2e" % (dtype, mode, banded, rel))
    assert rel < (1e-6 if dtype == torch.float64 else 2e-3), (rel, torch.isnan(zr).any(1).tolist(), torch.isnan(zp).any(1).tolist(), sr.tolist(), sp.tolist(), w.counts.tolist())
    (zp[:, :n] * wgt).sum().backward()
    gate = 1e-4 if dtype == torch.float64 else 1e-3                               # DESIGN.md section 5
    pairs = [(vr.grad, vp.grad[:, :n])] + [(geo[k].grad, geo2[k].grad) for k in geo]
    errs = {k: float((gr - gp).abs().max()) / max(1.0, float(gp.abs().max())) for k, (gr, gp) in zip(["v"] + list(geo), pairs)}
    print("gradient differences (dtype %s, mode %d, banded %s, exact %s): %s" % (dtype, mode, banded, exact, errs))
    assert max(errs.values()) < gate, errs


# ---------------------------------------------------------------------------------------------------- world_large replay
def test_world_large_replay_with_floor_as_obstacle():
    """world_large.npz: 60 circles on a pinned reference `Rect` floor (body 0, pinned by Je, body1 of every floor
    contact). Dropping the floor's dofs and Je and turning its contacts into one-body contacts (circle as body1,
    normal negated, p1 <-> p2) reproduces the reference's 16 engine results for the circles."""
    from lcp_physics_b200.engines import engine_solve
    recs = load_world_records("world_large")
    assert len(recs) >= 16
    worst, floor_contacts = 0.0, []
    for rec in recs:
        t = lambda k: torch.from_numpy(np.asarray(rec[k])).double().cuda()
        Je = np.asarray(rec["Je"])
        assert Je.shape[0] == 3 and np.array_equal(Je[:, :3], np.eye(3)) and not Je[:, 3:].any()
        Md = torch.diagonal(t("M"))
        nb = Md.numel() // 3 - 1
        inertia, mass = Md[3::3].unsqueeze(0), Md[4::3].unsqueeze(0)
        b1, b2 = np.asarray(rec["b1"]).astype(np.int64), np.asarray(rec["b2"]).astype(np.int64)
        nrm, p1, p2 = t("normal"), t("p1"), t("p2")
        fl = torch.from_numpy(b1 == 0).cuda()
        assert not (b2 == 0).any()
        floor_contacts.append(int(fl.sum()))
        nb1 = np.where(b1 == 0, b2 - 1, b1 - 1)
        nb2 = np.where(b1 == 0, nb, b2 - 1)
        f = lambda c: c.unsqueeze(1)
        normal = torch.where(f(fl), -nrm, nrm)
        q1, q2 = torch.where(f(fl), p2, p1), torch.where(f(fl), p1, p2)
        fr, re = np.asarray(rec["fric"]), np.asarray(rec["rest"])
        mu = torch.from_numpy(0.5 * (fr[b1] + fr[b2])).cuda().unsqueeze(0)
        rest = torch.from_numpy(0.5 * (re[b1] + re[b2])).cuda().unsqueeze(0)
        i32 = lambda a: torch.from_numpy(a).to(torch.int32).cuda()
        sd = str(rec["kind"]) == "solve_dynamics"
        z, st = engine_solve(mass, inertia, t("v")[3:].unsqueeze(0), t("f")[3:].unsqueeze(0), normal.unsqueeze(0),
                             q1.unsqueeze(0), q2.unsqueeze(0), mu, rest, i32(nb1), i32(nb2),
                             float(rec["dt"]) if sd else 0.0, mode=0 if sd else 1)
        ref = torch.from_numpy(np.asarray(rec["result"])).reshape(-1)[3:]
        out = (-z).reshape(-1).cpu()
        worst = max(worst, float((out - ref).norm() / ref.norm().clamp_min(1.0)))
    assert floor_contacts[0] == 10, floor_contacts
    assert worst < 1e-6, worst


# ---------------------------------------------------------------------------------------------------- trajectories
@pytest.mark.parametrize("post_stab", [False, True])
def test_batched_world_with_obstacles_reproduces_reference(post_stab):
    z = np.load(GOLDEN)
    w = golden_world(z, post_stab=post_stab)
    tag = "ps" if post_stab else "nops"
    nb = z["pos"].shape[1]
    worst = 0.0
    for k in range(25):
        w.step()
        assert w.counts.cpu().tolist() == z[tag + "_nc"][k].tolist(), k
        assert np.abs(w.t.cpu().numpy() - z[tag + "_t"][k]).max() < 1e-12, k       # same dt-halving history
        worst = max(worst, float(np.abs(w.p.cpu().numpy() - z[tag + "_p"][k][:, :nb]).max()))
    assert worst < 1e-6, worst


def test_large_pile_in_bin_matches_obstacle_oracle():
    """150 balls (n = 450 > 128: banded kernel) in a bin of 6 obstacles -- 6 pinned balls would not fit the banded
    kernel's 16-row border -- against the CPU oracle in the reference's pinned formulation."""
    from lcp_physics_b200.world import BatchedWorld
    from oracle.obstacle_oracle import OracleObstacleWorld
    sc = bin_scene(1, 150, 15, seed=3)
    nb = 150
    obst = sc["obst"]
    w = BatchedWorld(sc["pos"], sc["rad"], gravity=100.0, dt=1.0 / 30, obstacles=obst,
                     obstacle_fric=0.6, obstacle_rest=0.3, restitution=0.4, fric_coeff=0.5)
    assert w.large and w.no == 6
    orc = OracleObstacleWorld(sc["pos"][0], sc["rad"][0], torch.zeros(nb, 3), torch.ones(nb), torch.full((nb,), 0.4),
                              torch.full((nb,), 0.5), list(obst), obstacle_fric=0.6, obstacle_rest=0.3, gravity=100.0)
    assert int(w.counts[0]) == len(orc.contacts)
    assert int((w.c_b2[0, :int(w.counts[0])] >= nb).sum()) > 20                   # floor + walls touch many balls
    for k in range(3):
        w.step()
        orc.step()
        assert int(w.counts[0]) == len(orc.contacts), k
        err = float((w.p[0].cpu() - orc.p[:nb]).abs().max())
        assert err < 1e-6, (k, err)


def _pad(v, V):
    """Repeat-free padding of a convex polygon to V vertices: split its longest edges at their midpoints."""
    v = v.clone()
    while v.shape[0] < V:
        e = torch.roll(v, -1, 0) - v
        i = int(e.norm(dim=1).argmax())
        v = torch.cat([v[:i + 1], (v[i] + 0.5 * e[i]).unsqueeze(0), v[i + 1:]])
    return v


# ---------------------------------------------------------------------------------------------------- gradients
def test_ramp_rollout_gradients_match_central_differences():
    """A ball sliding down a ramp: d(final x) / d(ramp angle) and d(final x) / d(ball friction) through 8 steps with
    exact_adjoint=True, against central differences (every solve converged)."""
    from lcp_physics_b200.engines import last_solve_info
    from lcp_physics_b200.world import BatchedWorld, rect_vertices
    rad = 10.0

    def rollout(angle, fric):
        c, s = torch.cos(angle), torch.sin(angle)                   # the ball rests on the ramp, 0.03 above it
        ctr = torch.tensor([200.0, 300.0], dtype=torch.float64, device="cuda")
        start = ctr + torch.stack([c * -20.0 + 5.0 * s, s * -20.0 - 5.0 * c]) + (rad + 0.03) * torch.stack([s, -c])
        verts = rect_vertices(ctr, torch.tensor([200.0, 10.0], dtype=torch.float64, device="cuda"), angle)
        w = BatchedWorld(start.reshape(1, 1, 2), rad, gravity=100.0, dt=1.0 / 60, obstacles=verts.unsqueeze(0),
                         obstacle_fric=0.2, obstacle_rest=0.0, restitution=0.0, fric_coeff=fric.reshape(1, 1),
                         exact_adjoint=True)
        for _ in range(8):
            w.step()
            assert bool((last_solve_info()["status"] == 2).all())
        return w.p[0, 0, 1]

    a0 = torch.tensor(0.35, dtype=torch.float64, device="cuda", requires_grad=True)
    f0 = torch.tensor(0.1, dtype=torch.float64, device="cuda", requires_grad=True)
    x = rollout(a0, f0)
    ga, gf = torch.autograd.grad(x, (a0, f0))
    with torch.no_grad():
        ha, hf = 1e-5, 1e-5
        fa = (rollout(a0 + ha, f0) - rollout(a0 - ha, f0)) / (2 * ha)
        ff = (rollout(a0, f0 + hf) - rollout(a0, f0 - hf)) / (2 * hf)
    for g, fd in ((ga, fa), (gf, ff)):
        assert abs(float(g) - float(fd)) <= 2e-3 * max(abs(float(fd)), 1e-3), (float(g), float(fd))
