"""GPU: constraints between bodies, no-contact pairs and time-dependent external forces in BatchedWorld
(`constraints=`, `no_contact=`, `external_force=`): the recorded reference engine calls with two-body equality rows
replayed through engine_solve and B200PdipmEngine, the trajectories recorded from the unmodified reference
(tests/golden/bworld_joints.npz), a batch of seeded chains against the joint oracle (oracle/joint_oracle.py), the masked
contact walk (lcpb200_contacts with no_contact) against the unmasked one, rollout gradients against central differences,
fp32 against fp64, the large-scene kernel with a joint, and the constructor checks."""
import ctypes
import os
import types

import numpy as np
import pytest
import torch

from oracle.joint_oracle import OracleJointWorld
from tests.test_gpu_polygons import polygon_walk, random_scene
from tests.test_joint_oracle import constraint_list

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bworld_joints.npz")
SCENES = ("chain", "fixed", "inference")
f64 = torch.float64


def specs(cons):
    """BatchedWorld constraint specs from the oracle's tuples"""
    from lcp_physics_b200.world import FixedJoint, Joint, RotConstraint, XConstraint, YConstraint
    out = []
    for c in cons:
        if c[0] == "joint":
            out.append(Joint(c[1], c[2], c[3]))
        elif c[0] == "fixed":
            out.append(FixedJoint(c[1], c[2]))
        else:
            out.append({"x": XConstraint, "y": YConstraint, "rot": RotConstraint}[c[0]](c[1]))
    return out


def impulse(mult, nd, threshold=0.1):
    """forces.py hor_impulse(t) * multiplier [B] on body 0 (the projectile), per scene"""
    def f(t):
        out = torch.zeros(t.shape[0], nd, 3, dtype=t.dtype, device=t.device)
        out[:, 0, 1] = torch.where(t < threshold, mult.to(t.dtype), torch.zeros_like(t))
        return out
    return f


def golden_world(z, scene, dtype=f64, **kw):
    """BatchedWorld of a recorded scene: circles, the Rects as polygons, the pinned Rects as obstacles"""
    from lcp_physics_b200.world import BatchedWorld
    g = lambda k: torch.from_numpy(z["%s_%s" % (scene, k)])
    nc, ns = int(z[scene + "_ncirc"]), int(z[scene + "_nstatic"])
    p, v, m, fr, rs, hv = (g("init_" + k) for k in ("p", "v", "mass", "fric", "rest", "verts"))
    B, nbod = p.shape[0], p.shape[1]
    nr = nbod - nc - ns
    nd = nc + nr
    wv = hv + p[:, nc:, None, 1:]                                                   # world frame
    ob = dict(obstacles=wv[:, nr:], obstacle_fric=fr[:, nd:], obstacle_rest=rs[:, nd:]) if ns else {}
    mult = g("force")
    ext = impulse(mult.cuda(), nd) if float(mult.abs().max()) > 0 else None
    gm = [False] * nc + z[scene + "_gravity"][0].tolist()
    w = BatchedWorld(p[:, :nc, 1:].to(dtype), g("rad"), vel=v[:, :nc], mass=m[:, :nc], restitution=rs[:, :nc],
                     fric_coeff=fr[:, :nc], gravity=100.0, gravity_mask=gm, dt=1.0 / 30,
                     post_stab=bool(z[scene + "_post_stab"]), polygons=wv[:, :nr], poly_rot=p[:, nc:nd, 0],
                     poly_vel=v[:, nc:nd], poly_mass=m[:, nc:nd], poly_fric=fr[:, nc:nd], poly_rest=rs[:, nc:nd],
                     constraints=specs(constraint_list(z, scene, 0)),
                     no_contact=[(nc + int(a), nc + int(b)) for a, b in z[scene + "_no_contact"][0]],
                     external_force=ext, device="cuda", **ob, **kw)
    return w, nd


def check_converged(w):
    """wraps w._lcp: every solve of the rollout must converge (status 2, residual < 1e-8)"""
    from lcp_physics_b200.engines import last_solve_info
    orig = w._lcp

    def lcp(*a, **k):
        z = orig(*a, **k)
        info = last_solve_info()
        assert bool((info["status"] == 2).all()) and float(info["resid"].max()) < 1e-8, (
            info["status"].tolist(), float(info["resid"].max()))
        return z
    w._lcp = lcp
    return w


# ---------------------------------------------------------------------------------------------------- engine replay
def _calls(z, scene):
    for k in range(z[scene + "_call_mode"].shape[0]):
        g = lambda key: z["%s_call_%s" % (scene, key)][k]
        n = int(z[scene + "_call_n"][k])
        yield (int(g("mode")), float(g("dt")), g("Md"), g("v"), g("f"), g("normal")[:n], g("p1")[:n], g("p2")[:n],
               g("b1")[:n], g("b2")[:n], g("mu")[:n], g("rest")[:n], g("Je"), g("ge"), g("out"))


@pytest.mark.parametrize("exact", [False, True])
def test_engine_replay_with_two_body_equality_rows(exact):
    """The reference's engine calls (joints' rows in Je, b = 0 / Je v) through engine_solve: <= 1e-6 relative."""
    from lcp_physics_b200.engines import engine_solve
    z = np.load(GOLDEN)
    worst, seen = 0.0, set()
    for scene in SCENES:
        for mode, dt, Md, v, f, nrm, p1, p2, b1, b2, mu, rest, Je, ge, out in _calls(z, scene):
            c = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda().unsqueeze(0)
            i32 = lambda a: torch.from_numpy(a.astype(np.int32)).cuda()
            Mb = Md.reshape(-1, 3)
            zhat, status = engine_solve(c(Mb[:, 1]), c(Mb[:, 0]), c(v), c(f), c(nrm), c(p1), c(p2), c(mu), c(rest),
                                        i32(b1), i32(b2), dt, A=c(Je), b=c(ge), mode=mode, max_iter=10,
                                        exact_adjoint=exact)
            assert int(status[0]) != -100
            err = float((-zhat[0].cpu() - torch.from_numpy(out)).abs().max()) / max(1.0, float(np.abs(out).max()))
            worst = max(worst, err)
            seen.add((scene, mode))
    assert worst <= 1e-6, worst
    assert {("chain", 1), ("fixed", 0), ("inference", 0), ("inference", 1)} <= seen


def test_engine_replay_through_b200_pdipm_engine():
    """The same calls through B200PdipmEngine's fused path, from a stand-in World (the engine reads M(), Je(),
    get_v(), apply_forces(t), contacts and the bodies' materials)."""
    from lcp_physics_b200.engines import B200PdipmEngine
    z = np.load(GOLDEN)
    eng = B200PdipmEngine()
    worst = 0.0
    for scene in SCENES:
        fr, rs = z[scene + "_init_fric"][0], z[scene + "_init_rest"][0]
        bodies = [types.SimpleNamespace(fric_coeff=float(a), restitution=float(b)) for a, b in zip(fr, rs)]
        for mode, dt, Md, v, f, nrm, p1, p2, b1, b2, mu, rest, Je, ge, out in _calls(z, scene):
            t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
            cs = [((t(nrm[k]), t(p1[k]), t(p2[k]), torch.tensor(0.0, dtype=f64)), int(b1[k]), int(b2[k]))
                  for k in range(len(b1))]
            w = types.SimpleNamespace(t=0.0, bodies=bodies, contacts=cs, vec_len=3, static_inverse=False,
                                      fric_dirs=2, M=lambda: torch.diag(t(Md)), Je=lambda: t(Je),
                                      apply_forces=lambda _t: t(f), get_v=lambda: t(v))
            got = eng.solve_dynamics(w, dt) if mode == 0 else eng.post_stabilization(w).reshape(-1)
            worst = max(worst, float((got.cpu() - t(out)).abs().max()) / max(1.0, float(np.abs(out).max())))
    assert worst <= 1e-6, worst


# ---------------------------------------------------------------------------------------------------- trajectories
@pytest.mark.parametrize("exact", [False, True])
@pytest.mark.parametrize("scene", SCENES)
def test_batched_world_with_joints_reproduces_reference(scene, exact):
    z = np.load(GOLDEN)
    w, nd = golden_world(z, scene, exact_adjoint=exact)
    worst = 0.0
    for k in range(z[scene + "_nc"].shape[0]):
        w.step()
        assert w.counts.cpu().tolist() == z[scene + "_nc"][k].tolist(), k
        assert np.abs(w.t.cpu().numpy() - z[scene + "_t"][k]).max() < 1e-12, k        # same dt-halving history
        worst = max(worst, float(np.abs(w.p.cpu().numpy() - z[scene + "_p"][k][:, :nd]).max()))
    assert worst < 1e-6, worst


def test_fp32_joint_rollout_agrees_with_fp64():
    """fixed_joint_demo's welded boxes landing on the ramp, 20 steps in fp32 against fp64"""
    z = np.load(GOLDEN)
    w64, _ = golden_world(z, "fixed")
    w32, _ = golden_world(z, "fixed", dtype=torch.float32)
    assert w32.dtype == torch.float32 and w32.A.dtype == torch.float32
    for _ in range(20):
        w64.step()
        w32.step()
    d = (w32.p.double() - w64.p).abs()
    print("fp32 vs fp64 after 20 steps: position %.3e, rotation %.3e" % (float(d[..., 1:].max()), float(d[..., 0].max())))
    assert float(d[..., 1:].max()) < 1e-2 and float(d[..., 0].max()) < 1e-3, (float(d[..., 1:].max()),
                                                                            float(d[..., 0].max()))


# ---------------------------------------------------------------------------------------------------- batch
def chain_batch(B, seed, nl=4, steps_apart=True):
    """B pendulum chains: link 0 hung from a world point, nl - 1 link joints (neighbours excluded from contact),
    per-scene anchor, link dims and masses, and a circle moving at the last link"""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.rand(*s, generator=g, dtype=f64)
    ax = 300.0 + 10.0 * (r(B) - 0.5)
    dims = torch.stack([16.0 + 8.0 * r(B), 50.0 + 10.0 * r(B)], 1)                 # [B, 2], shared by a scene's links
    mass = 0.5 + r(B, nl)
    return dict(ax=ax, dims=dims, mass=mass, nl=nl, cy=lambda k: 50.0 + 50.0 * k, B=B)


def chain_world(sc, dtype=f64, **kw):
    from lcp_physics_b200.world import BatchedWorld, Joint, rect_vertices
    B, nl = sc["B"], sc["nl"]
    verts = torch.stack([torch.stack([rect_vertices(torch.stack([sc["ax"][b], torch.tensor(sc["cy"](k), dtype=f64)]),
                                                    sc["dims"][b]) for k in range(nl)]) for b in range(B)])
    anchors = torch.stack([sc["ax"], torch.full((B,), sc["cy"](0) - 20.0, dtype=f64)], 1)
    cons = [Joint(1, None, anchors)] + [Joint(1 + k, k, [float(sc["ax"][0]), sc["cy"](k) - 25.0]) for k in range(1, nl)]
    # each scene's link joints at its own anchor x
    for k in range(1, nl):
        cons[k].anchor = torch.stack([sc["ax"], torch.full((B,), sc["cy"](k) - 25.0, dtype=f64)], 1)
    cpos = torch.stack([sc["ax"] - sc["dims"][:, 0] / 2 - 12.0 - 3.0, torch.full((B,), sc["cy"](nl - 1), dtype=f64)], 1)
    w = BatchedWorld(cpos.unsqueeze(1).to(dtype), 10.0, vel=torch.tensor([0.0, 60.0, 0.0]).expand(B, 1, 3),
                     gravity=100.0, gravity_mask=[False] + [True] * nl, dt=1.0 / 30, polygons=verts,
                     poly_mass=sc["mass"], constraints=cons, no_contact=[(1 + k, k) for k in range(1, nl)],
                     device="cuda", **kw)
    return w, verts, anchors, cons


def chain_oracle(sc, w, verts, cons, b):
    """the joint oracle of scene b of chain_world"""
    from lcp_physics_b200.world import polygon_centroid
    nl = sc["nl"]
    cen = polygon_centroid(verts[b])
    hp = torch.cat([torch.zeros(nl, 1, dtype=f64), cen], 1)
    oc = [("joint", c.i, c.j, c.anchor[b].tolist()) for c in cons]
    return OracleJointWorld(w.p[b, :1, 1:].cpu(), [10.0], w.v[b, :3].cpu(), [1.0], [0.5], [0.9],
                            [v - c for v, c in zip(verts[b], cen)], hp, torch.zeros(nl, 3), sc["mass"][b],
                            w.inertia[b, 1:].cpu(), [0.9] * nl, [0.5] * nl, [True] * nl, gravity=100.0, dt=1.0 / 30,
                            constraints=oc, no_contact=[(1 + k, k) for k in range(1, nl)],
                            gravity_mask=[False] + [True] * nl)


def test_batch_of_seeded_chains_matches_joint_oracle():
    """256 chains with per-scene anchors, link dims and masses, each hit by a circle, against the oracle"""
    sc = chain_batch(256, 11)
    w, verts, anchors, cons = chain_world(sc)
    picked = list(range(0, 256, 16)) + [255]
    orcs = {b: chain_oracle(sc, w, verts, cons, b) for b in picked}
    hits = 0
    for k in range(10):
        w.step()
        for b, o in orcs.items():
            o.step()
            assert int(w.counts[b]) == len(o.contacts), (k, b)
            assert abs(float(w.t[b]) - o.t) < 1e-12
            err = float((w.p[b].cpu() - o.p).abs().max())
            assert err < 1e-6, (k, b, err)
        hits += int((w.counts > 0).sum())
    assert hits > 0


# ---------------------------------------------------------------------------------------------------- masked walk
def mask_walk(scs, dtype, cap, excl):
    """lcpb200_contacts with no_contact (the mask walk) on scenes of equal shapes with the pairs `excl` excluded"""
    from lcp_physics_b200 import _lib
    from lcp_physics_b200.world import polygon_centroid
    lib = _lib.load()
    B = len(scs)
    st = lambda k: torch.stack([s[k] for s in scs]).to("cuda", dtype).contiguous()
    pos, rad, pv, ov = st("pos"), st("rad"), st("polys"), st("obst")
    nb, npoly, no = pos.shape[1], pv.shape[1], ov.shape[1]
    nt = nb + npoly + no
    pcen = polygon_centroid(pv).contiguous() if npoly else None
    oref = polygon_centroid(ov).contiguous() if no else None
    fr, rs = torch.full((B, nb), 0.5, dtype=dtype, device="cuda"), torch.zeros(B, nb, dtype=dtype, device="cuda")
    pfr, ofr = st("pfric"), st("ofric")
    prs, ors = torch.zeros_like(pfr), torch.zeros_like(ofr)
    words = np.zeros((nt * nt + 31) // 32, dtype=np.uint32)
    for a, b in excl:
        bit = a * nt + b
        words[bit >> 5] |= np.uint32(1 << (bit & 31))
    mask = torch.from_numpy(words.view(np.int32)).cuda()
    i32 = lambda *s: torch.empty(*s, dtype=torch.int32, device="cuda")
    b1, b2, feat, counts = i32(B, cap), i32(B, cap), i32(B, cap), i32(B)
    new = lambda *s: torch.empty(B, cap, *s, dtype=dtype, device="cuda")
    geo = [new(2), new(2), new(2), new(), new(), new()]
    _lib.check(lib.lcpb200_contacts(
        _lib.dtype_code(dtype), B, nb, npoly, no, 6, cap, 0.1,
        *[_lib.ptr(t) for t in (pos, rad, fr, rs, pv, pcen, pfr, prs, ov, oref, ofr, ors, b1, b2, counts, feat)],
        *[_lib.ptr(t) for t in geo], _lib.ptr(mask), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    return dict(b1=b1, b2=b2, feat=feat, counts=counts, geo=geo)


@pytest.mark.parametrize("sizes", [(14, 0, 0, 60.0), (12, 0, 3, 80.0), (3, 8, 2, 60.0), (10, 36, 4, 140.0)])
def test_mask_walk_equals_polygon_walk_without_excluded_pairs(sizes):
    """circles only, circles + obstacles, mixed polygon scenes (the last spans two 1024-pair chunks): the masked walk
    gives the unmasked walk's contacts minus the excluded pairs, in the same order, with the same feat and bitwise
    equal geometry"""
    nc, npoly, no, spread = sizes
    scs = [random_scene(100 + s, nc, npoly, no, spread) for s in range(4)]
    full = polygon_walk(scs, f64, cap=1024)
    nd, nt = nc + npoly, nc + npoly + no
    pairs = set()
    for s in range(4):                                        # exclude about half of the pairs that make contact
        n = int(full["counts"][s])
        pairs |= {(int(a), int(b)) for a, b in zip(full["b1"][s, :n].tolist(), full["b2"][s, :n].tolist())}
    excl = sorted(pairs)[::2] + [(nd, nt - 1)] if no > 1 else sorted(pairs)[::2]   # + an obstacle-obstacle pair
    got = mask_walk(scs, f64, 1024, excl)
    ex = set(excl)
    removed = 0
    for s in range(4):
        n = int(full["counts"][s])
        keep = [k for k in range(n) if (int(full["b1"][s, k]), int(full["b2"][s, k])) not in ex]
        removed += n - len(keep)
        m = int(got["counts"][s])
        assert m == len(keep), (s, m, len(keep))
        idx = torch.tensor(keep, dtype=torch.long, device="cuda")
        for key in ("b1", "b2", "feat"):
            assert torch.equal(got[key][s, :m], full[key][s].index_select(0, idx)), (s, key)
        for a, b in zip(got["geo"], full["geo"]):
            assert torch.equal(a[s, :m], b[s].index_select(0, idx)), s
    assert removed > 0


@pytest.mark.parametrize("with_obstacles", [False, True])
def test_no_contact_world_matches_find_contacts_torch(with_obstacles):
    """polygon-free BatchedWorld with no_contact: the masked walk's list equals find_contacts_torch's"""
    from lcp_physics_b200.world import BatchedWorld, rect_vertices
    g = torch.Generator().manual_seed(5)
    B, nb = 8, 24
    pos = torch.rand(B, nb, 2, generator=g, dtype=f64) * 60.0
    ob = dict(obstacles=torch.stack([rect_vertices([30.0, 70.0], [80.0, 10.0]),
                                     rect_vertices([30.0, -8.0], [80.0, 10.0], 0.1)])) if with_obstacles else {}
    excl = [(0, 1), (2, 5), (3, 7), (1, 10)] + ([(4, nb), (6, nb + 1), (nb, nb + 1)] if with_obstacles else [])
    w = BatchedWorld(pos, 4.0, no_contact=excl, strict_no_penetration=False, device="cuda", contact_capacity=256, **ob)
    counts, b1, b2 = w.find_contacts_torch()
    assert torch.equal(counts, w.counts)
    for s in range(B):
        n = int(counts[s])
        assert torch.equal(b1[s, :n], w.c_b1[s, :n]) and torch.equal(b2[s, :n], w.c_b2[s, :n]), s
        assert not any((a, b) in set(excl) for a, b in zip(b1[s, :n].tolist(), b2[s, :n].tolist()))
    plain = BatchedWorld(pos, 4.0, strict_no_penetration=False, device="cuda", contact_capacity=256, **ob)
    assert int(plain.counts.sum()) > int(w.counts.sum())


# ---------------------------------------------------------------------------------------------------- gradients
def _fd_check(rollout, leaves, h, history=None):
    """analytic gradients of rollout(*leaves) against central differences with steps h; max |diff| / FD scale.
    history (a list the rollout appends its step history to): every FD rollout must take the same steps (dt halvings,
    contact counts) as the base rollout, or the difference straddles a discontinuity"""
    y = rollout(*leaves)
    grads = torch.autograd.grad(y, leaves)
    fds, gs = [], []
    with torch.no_grad():
        for k in range(len(leaves)):
            for comp in range(leaves[k].numel()):
                plus = [t.detach().clone() for t in leaves]
                minus = [t.detach().clone() for t in leaves]
                plus[k].view(-1)[comp] += h[k]
                minus[k].view(-1)[comp] -= h[k]
                fds.append(float((rollout(*plus) - rollout(*minus)) / (2 * h[k])))
                gs.append(float(grads[k].reshape(-1)[comp]))
                if history is not None:
                    assert history[-1] == history[0] and history[-2] == history[0], (k, history[0], history[-2:])
    scale = max(abs(f) for f in fds)
    err = max(abs(a - b) for a, b in zip(gs, fds)) / scale
    return err, gs, fds


def test_pendulum_chain_gradients_match_central_differences():
    """(a) a contact-free chain (world anchor + 4 links, gravity): final link positions w.r.t. the link mass, the
    anchor's x and link 0's initial angular velocity, exact_adjoint=True"""
    from lcp_physics_b200.world import BatchedWorld, Joint, rect_vertices
    dev = "cuda"

    def rollout(mass, ax, w0):
        verts = torch.stack([rect_vertices(torch.stack([torch.tensor(300.0, dtype=f64, device=dev),
                                                        torch.tensor(50.0 + 50.0 * k, dtype=f64, device=dev)]),
                                           torch.tensor([20.0, 60.0], dtype=f64, device=dev)) for k in range(4)])
        vel = torch.zeros(1, 4, 3, dtype=f64, device=dev)
        vel = vel + torch.nn.functional.pad(w0.reshape(1, 1, 1), (0, 2, 0, 3))
        anchor = torch.stack([ax, torch.tensor(25.0, dtype=f64, device=dev)])
        cons = [Joint(0, None, anchor)] + [Joint(k, k - 1, [300.0, 25.0 + 50.0 * k]) for k in range(1, 4)]
        w = BatchedWorld(torch.zeros(1, 0, 2, dtype=f64, device=dev), 1.0, gravity=100.0, dt=1.0 / 30,
                         polygons=verts.unsqueeze(0), poly_vel=vel, poly_mass=mass.expand(1, 4), constraints=cons,
                         no_contact=[(k, k - 1) for k in range(1, 4)], exact_adjoint=True, device=dev)
        check_converged(w)
        for _ in range(10):
            w.step()
            assert int(w.counts.max()) == 0
        return (w.p[0, :, 1:] * torch.tensor([1.0, 0.5], dtype=f64, device=dev)).sum() + 10.0 * w.p[0, :, 0].sum()

    leaves = [torch.tensor(v, dtype=f64, device=dev).requires_grad_(True) for v in (1.3, 300.5, 0.2)]
    err, gs, fds = _fd_check(rollout, leaves, [1e-5, 1e-4, 1e-6])
    print("pendulum chain: analytic %s, central differences %s, max |diff| / FD scale %.2e" % (gs, fds, err))
    assert err < 1e-4, (err, gs, fds)


def test_inference_chain_gradients_match_central_differences():
    """(b) inference.py's chain (world anchor, 10 links, a restitution-1 projectile under hor_impulse) with friction 0:
    link positions after the hit w.r.t. the chain's mass and the impulse multiplier, exact_adjoint=True"""
    from lcp_physics_b200.world import BatchedWorld, Joint, rect_vertices
    dev = "cuda"
    verts = torch.stack([rect_vertices([300.0, 50.0 + 50.0 * k], [20.0, 60.0]) for k in range(10)]).to(dev)
    cons = [Joint(1, None, [300.0, 30.0])] + [Joint(1 + k, k, [300.0, 25.0 + 50.0 * k]) for k in range(1, 10)]

    history = []

    def rollout(total, mult):
        w = BatchedWorld(torch.tensor([[[200.0, 500.0]]], dtype=f64, device=dev), 20.0, restitution=1.0, fric_coeff=0.0,
                         gravity=100.0, gravity_mask=[False, False] + [True] * 9, dt=1.0 / 30, post_stab=True,
                         polygons=verts.unsqueeze(0), poly_mass=(total / 10).expand(1, 10), poly_fric=0.0,
                         constraints=cons, no_contact=[(1 + k, k) for k in range(1, 10)],
                         external_force=impulse(mult.reshape(1), 11), exact_adjoint=True, device=dev, tol=1e-4)
        check_converged(w)
        steps = []
        for _ in range(22):
            w.step()
            steps.append((float(w.t[0]), int(w.counts[0])))
        assert any(c > 0 for _, c in steps)
        history.append(steps)
        return (w.p[0, 1:, 1:] * torch.tensor([1.0, 0.3], dtype=f64, device=dev)).sum()

    leaves = [torch.tensor(v, dtype=f64, device=dev).requires_grad_(True) for v in (7.0, 1500.0)]
    err, gs, fds = _fd_check(rollout, leaves, [7e-6, 1.5e-3], history)
    print("inference chain: analytic %s, central differences %s, max |diff| / FD scale %.2e" % (gs, fds, err))
    assert err < 1e-4, (err, gs, fds)


# ---------------------------------------------------------------------------------------------------- large scene
def _large_pile(n=44):
    """n circles (radius 5) in two touching rows on a floor obstacle: 3 n > 128, the banded kernel"""
    from lcp_physics_b200.world import rect_vertices
    g = torch.Generator().manual_seed(3)
    xs = [60.0 + 10.02 * (k % 22) + 0.01 * float(torch.rand(1, generator=g)) for k in range(n)]
    ys = [495.0 - 0.03 - (k // 22) * 9.0 for k in range(n)]
    for k in range(22, n):
        xs[k] += 5.0
    return torch.tensor([xs, ys], dtype=f64).t().contiguous(), rect_vertices([200.0, 505.0], [400.0, 10.0])


def test_large_scene_with_a_joint_runs_on_banded_kernel_and_matches_oracle():
    from lcp_physics_b200.world import BatchedWorld, Joint, polygon_centroid
    pos, floor = _large_pile()
    n = pos.shape[0]
    anchor = ((pos[3] + pos[4]) / 2).tolist()
    w = BatchedWorld(pos.unsqueeze(0), 5.0, gravity=100.0, dt=1.0 / 30, obstacles=floor.unsqueeze(0),
                     constraints=[Joint(3, 4, anchor)], no_contact=[(3, 4)], device="cuda")
    assert w.large and w.ne == 2
    cen = polygon_centroid(floor)
    orc = OracleJointWorld(pos, torch.full((n,), 5.0), torch.zeros(n, 3), torch.ones(n), torch.full((n,), 0.5),
                           torch.full((n,), 0.9), [floor - cen], torch.cat([torch.zeros(1), cen]).reshape(1, 3),
                           torch.zeros(1, 3), torch.ones(1), [1.0], [0.9], [0.5], [True], n_static=1,
                           constraints=[("joint", 3, 4, anchor)], no_contact=[(3, 4)])
    assert int(w.counts[0]) == len(orc.contacts) > 0
    for k in range(3):
        w.step()
        orc.step()
        assert int(w.counts[0]) == len(orc.contacts), k
        err = float((w.p[0].cpu() - orc.p[:n]).abs().max())
        assert err < 1e-6, (k, err)


def test_large_scene_with_joints_overflowing_the_border_raises():
    from lcp_physics_b200.world import BatchedWorld, Joint
    pos, floor = _large_pile()
    cons = [Joint(k, k + 1, ((pos[k] + pos[k + 1]) / 2).tolist()) for k in range(3)]   # 3 x 4 bodies + 6 rows
    with pytest.raises(ValueError, match="border"):
        BatchedWorld(pos.unsqueeze(0), 5.0, obstacles=floor.unsqueeze(0), constraints=cons, device="cuda")


# ---------------------------------------------------------------------------------------------------- API
def test_constraint_api_errors():
    from lcp_physics_b200.world import BatchedWorld, FixedJoint, Joint, XConstraint, rect_vertices
    pos = torch.tensor([[[0.0, 0.0], [30.0, 0.0]]], dtype=f64)
    ob = dict(obstacles=rect_vertices([0.0, 40.0], [100.0, 10.0]).unsqueeze(0))
    mk = lambda **kw: BatchedWorld(pos, 5.0, device="cuda", **ob, **kw)
    with pytest.raises(ValueError, match="out of range"):
        mk(constraints=[XConstraint(5)])
    with pytest.raises(ValueError, match="obstacle"):
        mk(constraints=[Joint(0, 2, [0.0, 0.0])])
    with pytest.raises(ValueError, match="itself"):
        mk(constraints=[Joint(1, 1, [0.0, 0.0])])
    with pytest.raises(ValueError, match="non-finite"):
        mk(constraints=[Joint(0, 1, [float("nan"), 0.0])])
    with pytest.raises(ValueError, match="two bodies"):
        mk(constraints=[FixedJoint(0, None)])
    with pytest.raises(ValueError, match="no_contact: body index out of range"):
        mk(no_contact=[(0, 3)])
    with pytest.raises(ValueError, match="twice"):
        mk(no_contact=[(1, 1)])
    w = mk(no_contact=[(2, 0)], constraints=[Joint(0, 1, [15.0, 0.0]), XConstraint(0)],
           external_force=lambda t: torch.zeros(1, 2, 2, dtype=f64, device="cuda"))
    assert w.ne == 3 and w.A.shape == (1, 3, 6)
    with pytest.raises(ValueError, match="external_force"):
        w.step()
    plain = mk()
    assert plain.A is None and plain.nc_mask is None and plain.cons == []
