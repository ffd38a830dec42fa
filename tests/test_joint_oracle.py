"""CPU: the restatement of the reference `World.step_dt` with constraints between bodies, add_no_contact pairs and
time-dependent external forces (oracle/joint_oracle.py) against trajectories recorded from the unmodified reference
(tests/golden/bworld_joints.npz: chain_demo's chain hit by a projectile, fixed_joint_demo's welded boxes on a ramp,
inference.py's chain hung from a world point), and the constructor checks of BatchedWorld's constraint keywords."""
import os

import numpy as np
import pytest
import torch

from oracle.joint_oracle import OracleJointWorld

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bworld_joints.npz")
SCENES = ("chain", "fixed", "inference")
KINDS = {0: "x", 1: "y", 2: "rot", 3: "joint", 4: "fixed"}


def constraint_list(z, scene, w):
    """("joint", i, j, anchor) / ("fixed", i, j) / ("x", i) ... with body indices in [circles, polygons]"""
    nc = int(z[scene + "_ncirc"])
    out = []
    for (k, i, j), a in zip(z[scene + "_cons"][w], z[scene + "_anchor"][w]):
        kind = KINDS[int(k)]
        i, j = nc + int(i), None if j < 0 else nc + int(j)
        out.append((kind, i, j, a.tolist()) if kind == "joint" else (kind, i, j) if kind == "fixed" else (kind, i))
    return out


def hor_impulse(mult):
    """forces.py hor_impulse times the multiplier, on the circle (body 0) only; t is the reference's world.t"""
    def f(t, nd):
        out = torch.zeros(nd, 3, dtype=torch.float64)
        if t < 0.1:
            out[0, 1] = mult
        return out
    return f


def oracle_world(z, scene, w):
    g = lambda k: z["%s_%s" % (scene, k)][w]
    nc, ns = int(z[scene + "_ncirc"]), int(z[scene + "_nstatic"])
    p, v, m, inert, fr, rs = (g("init_" + k) for k in ("p", "v", "mass", "inertia", "fric", "rest"))
    nd = p.shape[0] - ns
    mult = float(g("force"))
    f = hor_impulse(mult) if mult != 0 else None
    gm = [False] * nc + list(g("gravity"))
    return OracleJointWorld(
        p[:nc, 1:], g("rad"), v[:nc], m[:nc], rs[:nc], fr[:nc], [torch.from_numpy(x) for x in g("init_verts")],
        p[nc:], v[nc:], m[nc:], inert[nc:], fr[nc:], rs[nc:], [True] * (p.shape[0] - nc), n_static=ns, gravity=100.0,
        dt=1.0 / 30, post_stab=bool(z[scene + "_post_stab"]), constraints=constraint_list(z, scene, w),
        no_contact=[(nc + int(a), nc + int(b)) for a, b in g("no_contact")], gravity_mask=gm,
        force=(lambda t: f(t, nd)) if f else None)


@pytest.mark.parametrize("scene", SCENES)
def test_joint_oracle_matches_reference_world(scene):
    z = np.load(GOLDEN)
    for w in range(z[scene + "_p"].shape[1]):
        world = oracle_world(z, scene, w)
        for k in range(z[scene + "_nc"].shape[0]):
            world.step()
            assert len(world.contacts) == int(z[scene + "_nc"][k, w]), (w, k)
            assert abs(world.t - z[scene + "_t"][k, w]) < 1e-12, (w, k)
            assert np.abs(world.p.numpy() - z[scene + "_p"][k, w]).max() < 1e-9, (w, k)
            assert np.abs(world.v.numpy().reshape(-1, 3) - z[scene + "_v"][k, w]).max() < 1e-8, (w, k)


@pytest.mark.parametrize("scene", SCENES)
def test_recorded_scenes_make_contact(scene):
    """every recorded scene has steps with contacts (the projectile reaches the chain, the boxes the ramp) and the
    recorded engine calls include both modes where post-stabilisation is on"""
    z = np.load(GOLDEN)
    assert (z[scene + "_nc"] > 0).any(0).all()
    modes = set(z[scene + "_call_mode"].tolist())
    assert modes == ({0, 1} if bool(z[scene + "_post_stab"]) else {0})

