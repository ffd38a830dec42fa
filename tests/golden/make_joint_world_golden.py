"""Records trajectories and engine calls of B independent UNMODIFIED reference `World`s (ode/pygame stubbed,
oracle/ref_shim.py) with CONSTRAINTS between bodies, `add_no_contact` pairs and time-dependent external forces, for
`BatchedWorld(constraints=, no_contact=, external_force=)` and oracle/joint_oracle.py to reproduce:

    python tests/golden/make_joint_world_golden.py        (build container only)

Bodies are listed [circles..., Rect links / boxes..., pinned Rect obstacles...] (the order BatchedWorld's pair walk
follows); the constraint list is the obstacles' TotalConstraints first, then the scene's constraints in the demo's
order. Three scenes, B worlds each with per-world jitter:
  * chain: demos/demo.py chain_demo: 10 Rect links (20 x 60) joined by 9 `Joint`s with add_no_contact between
    neighbours, XConstraint + YConstraint on the top link, Gravity(100) on links 1-9, a projectile circle (radius 20)
    under ExternalForce(hor_impulse, 2000), post_stab=True (chain_demo's clock circle is left out);
    the projectile starts at x = 200 instead of 50 (here and in `inference`), so it hits the chain within ten steps;
  * fixed: demos/fixed_joint_demo.py: two 60 x 60 Rects welded by a `FixedJoint` with add_no_contact, Gravity(100), on
    the pinned tilted Rect ramp (pi / 32); the boxes start a few pixels above the ramp instead of 400 px up, so they
    land within the recorded steps;
  * inference: experiments/inference.py's make_world: Joint(link 0, None, (300, 30)) and 9 link joints with
    add_no_contact, link mass = total / 10, Gravity(100) on links 1-9, a projectile (radius 20, restitution 1) level
    with the last link under ExternalForce(hor_impulse, 1500), post_stab=True.
Stored per scene: p, v of every body, the contact count and t after every step; the initial bodies; the constraint
parameters; and, for world 0, every engine call that had contacts (both modes): M's diagonal, v, f, the contact list,
Je, ge and the returned solution.
"""
import math
import os
import random
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_shim  # noqa: E402

ref_shim.install_world_stubs()
import lcp_physics.physics.engines as ref_engines  # noqa: E402
from lcp_physics.physics.bodies import Circle, Rect  # noqa: E402
from lcp_physics.physics.constraints import FixedJoint, Joint, TotalConstraint, XConstraint, YConstraint  # noqa: E402
from lcp_physics.physics.forces import ExternalForce, Gravity, hor_impulse  # noqa: E402
from lcp_physics.physics.world import World  # noqa: E402

ref_engines.LCPFunction = ref_shim.ReferenceLCPFunction
OUT = os.path.dirname(os.path.abspath(__file__))
B = 2
STEPS = {"chain": 50, "fixed": 40, "inference": 60}
MAX_CALLS = 40


def chain_scene(seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda: float(torch.rand(1, generator=g))
    links = [((300.0, 50.0 + 50.0 * i), (20.0, 60.0), 1.0 + 0.2 * (r() - 0.5)) for i in range(10)]
    cons = [("x", 0), ("y", 0)] + [("joint", i, i - 1, (300.0, 25.0 + 50.0 * i)) for i in range(1, 10)]
    return dict(circles=[((200.0, 500.0 + 20.0 * (r() - 0.5)), 20.0, 1.0 + 0.2 * r())], rects=links, rest=0.9,
                fric=0.9, obstacles=[], cons=cons, no_contact=[(i, i - 1) for i in range(1, 10)],
                gravity=[False] + [True] * 9, force=("hor", 2000.0 * (1.0 + 0.1 * r())), post_stab=True)


def fixed_scene(seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda: float(torch.rand(1, generator=g))
    incl = math.pi / 32
    x0 = 120.0 + 10.0 * r()
    top = lambda x: 500.0 + (x - 500.0) * math.tan(incl) - 5.0 / math.cos(incl)    # the ramp's top edge
    y = top(x0 - 30.0) - 30.0 - 2.0 - 3.0 * r()          # the boxes' bottoms above the ramp's highest point below them
    rects = [((x0, y), (60.0, 60.0), 1.0), ((x0 + 40.0, y), (60.0, 60.0), 1.0 + 0.5 * r())]
    return dict(circles=[], rects=rects, rest=0.5, fric=0.15, obstacles=[((incl, 500.0, 500.0), (900.0, 10.0))],
                cons=[("fixed", 0, 1)], no_contact=[(1, 0)], gravity=[True, True], force=None, post_stab=False)


def inference_scene(seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda: float(torch.rand(1, generator=g))
    m = (7.0 + 2.0 * (r() - 0.5)) / 10
    links = [((300.0, 50.0 + 50.0 * i), (20.0, 60.0), m) for i in range(10)]
    cons = [("joint", 0, None, (300.0, 30.0))] + [("joint", i, i - 1, (300.0, 25.0 + 50.0 * i)) for i in range(1, 10)]
    return dict(circles=[((200.0, 500.0), 20.0, 1.0)], rects=links, rest=None, fric=None, circle_rest=1.0,
                obstacles=[], cons=cons, no_contact=[(i, i - 1) for i in range(1, 10)], gravity=[False] + [True] * 9,
                force=("hor", 500.0 * 3 * (1.0 + 0.1 * r())), post_stab=True)


def build(sc):
    """The reference World of a scene; body indices: circles, Rects, obstacles."""
    nc = len(sc["circles"])
    kw = lambda: {k: v for k, v in (("restitution", sc["rest"]), ("fric_coeff", sc["fric"])) if v is not None}
    bodies, rects = [], []
    for pos, rad, m in sc["circles"]:
        ck = kw()
        if "circle_rest" in sc:
            ck["restitution"] = sc["circle_rest"]
        c = Circle(list(pos), rad, mass=m, **ck)
        if sc["force"] is not None:
            c.add_force(ExternalForce(hor_impulse, multiplier=sc["force"][1]))
        bodies.append(c)
    for k, (pos, dims, m) in enumerate(sc["rects"]):
        o = Rect(list(pos), list(dims), mass=m, **kw())
        if sc["gravity"][k]:
            o.add_force(Gravity(g=100))
        bodies.append(o)
        rects.append(o)
    joints = []
    for pos, dims in sc["obstacles"]:
        o = Rect(list(pos), list(dims), **kw())
        joints.append(TotalConstraint(o))
        bodies.append(o)
    body = lambda k: rects[k]                          # constraints name the Rects by their index among the Rects
    for c in sc["cons"]:
        if c[0] == "x":
            joints.append(XConstraint(body(c[1])))
        elif c[0] == "y":
            joints.append(YConstraint(body(c[1])))
        elif c[0] == "fixed":
            joints.append(FixedJoint(body(c[1]), body(c[2])))
        else:
            joints.append(Joint(body(c[1]), None if c[2] is None else body(c[2]), list(c[3])))
    for a, b in sc["no_contact"]:
        rects[a].add_no_contact(rects[b])
    return World(bodies, joints, dt=1.0 / 30, post_stab=sc["post_stab"]), nc


def record_calls(world, calls):
    """Wraps world.engine's two methods to record every call that has contacts."""
    eng = world.engine

    def rec(mode, w, dt, out):
        if not w.contacts or len(calls) >= MAX_CALLS:
            return
        cs = w.contacts
        Je = w.Je()
        v = w.get_v()
        bodies = w.bodies
        calls.append(dict(
            mode=mode, dt=float(dt), Md=torch.diagonal(w.M()).detach().numpy().copy(), v=v.detach().numpy().copy(),
            f=(w.apply_forces(w.t) if mode == 0 else v.new_zeros(v.shape)).detach().numpy().copy(),
            normal=np.array([c[0][0].detach().numpy() for c in cs]), p1=np.array([c[0][1].detach().numpy() for c in cs]),
            p2=np.array([c[0][2].detach().numpy() for c in cs]), b1=np.array([c[1] for c in cs]),
            b2=np.array([c[2] for c in cs]),
            mu=np.array([0.5 * float(bodies[c[1]].fric_coeff + bodies[c[2]].fric_coeff) for c in cs]),
            rest=np.array([0.5 * float(bodies[c[1]].restitution + bodies[c[2]].restitution) for c in cs]),
            Je=Je.detach().numpy().copy(),
            ge=(torch.matmul(Je, v) if mode == 1 else Je.new_zeros(Je.shape[0])).detach().numpy().copy(),
            out=out.detach().reshape(-1).numpy().copy()))

    sd, ps = eng.solve_dynamics, eng.post_stabilization

    def solve_dynamics(w, dt):
        out = sd(w, dt)
        rec(0, w, dt, out)
        return out

    def post_stabilization(w):
        out = ps(w)
        rec(1, w, 0.0, out)
        return out

    eng.solve_dynamics, eng.post_stabilization = solve_dynamics, post_stabilization


def initial_bodies(world, nc):
    """The bodies as the reference holds them: p [nbodies, 3], v, mass, M[0, 0], friction, restitution, and the
    Rects' vertices about their centroid (Hull.verts)."""
    bs = world.bodies
    return dict(p=np.stack([b.p.detach().numpy() for b in bs]), v=np.stack([b.v.detach().numpy() for b in bs]),
                mass=np.array([float(b.mass) for b in bs]), inertia=np.array([float(b.M[0, 0]) for b in bs]),
                fric=np.array([float(b.fric_coeff) for b in bs]), rest=np.array([float(b.restitution) for b in bs]),
                verts=np.stack([torch.stack(list(b.verts)).detach().numpy() for b in bs[nc:]]))


def run(sc, steps, calls=None):
    world, nc = build(sc)
    init = initial_bodies(world, nc)
    if calls is not None:
        record_calls(world, calls)
    P, Vv, NC, T = [], [], [], []
    for _ in range(steps):
        world.step()
        P.append(torch.stack([b.p for b in world.bodies]).detach().numpy().copy())
        Vv.append(world.v.detach().numpy().reshape(-1, 3).copy())
        NC.append(len(world.contacts))
        T.append(float(world.t))
    return np.stack(P), np.stack(Vv), np.array(NC), np.array(T), init


def scene_arrays(sc):
    """The scene's parameters as arrays (what BatchedWorld and the oracle are built from)."""
    cons = sc["cons"]
    kind = {"x": 0, "y": 1, "rot": 2, "joint": 3, "fixed": 4}
    ci = np.array([[kind[c[0]], c[1], -1 if len(c) < 3 or c[2] is None else c[2]] for c in cons], dtype=np.int64)
    anchor = np.array([c[3] if c[0] == "joint" else (0.0, 0.0) for c in cons], dtype=np.float64)
    return dict(rad=np.array([c[1] for c in sc["circles"]]), rect_dims=np.array([r[1] for r in sc["rects"]]),
                obst=np.array([list(o[0]) + list(o[1]) for o in sc["obstacles"]]).reshape(-1, 5), cons=ci,
                anchor=anchor, no_contact=np.array(sc["no_contact"], dtype=np.int64).reshape(-1, 2),
                gravity=np.array(sc["gravity"]), force=np.array(sc["force"][1] if sc["force"] else 0.0))


def main():
    random.seed(0)
    torch.manual_seed(0)
    blob = {}
    for si, (name, make) in enumerate((("chain", chain_scene), ("fixed", fixed_scene),
                                       ("inference", inference_scene))):
        scenes = [make(500 + 31 * k + 1000 * si) for k in range(B)]
        sc0 = scenes[0]
        blob[name + "_post_stab"] = np.array(sc0["post_stab"])
        blob[name + "_ncirc"] = np.array(len(sc0["circles"]))
        blob[name + "_nstatic"] = np.array(len(sc0["obstacles"]))
        for key in scene_arrays(sc0):
            blob["%s_%s" % (name, key)] = np.stack([scene_arrays(sc)[key] for sc in scenes])
        calls = []
        res = [run(sc, STEPS[name], calls if k == 0 else None) for k, sc in enumerate(scenes)]
        for key, col in (("p", 0), ("v", 1), ("nc", 2), ("t", 3)):
            blob["%s_%s" % (name, key)] = np.stack([r[col] for r in res], 1)     # [steps, B, ...]
        for key in res[0][4]:
            blob["%s_init_%s" % (name, key)] = np.stack([r[4][key] for r in res])    # [B, ...]
        C = max(len(c["b1"]) for c in calls)
        blob[name + "_call_n"] = np.array([len(c["b1"]) for c in calls])
        for key in ("mode", "dt"):
            blob["%s_call_%s" % (name, key)] = np.array([c[key] for c in calls])
        for key in ("Md", "v", "f", "Je", "ge", "out"):
            blob["%s_call_%s" % (name, key)] = np.stack([c[key] for c in calls])
        for key in ("normal", "p1", "p2", "b1", "b2", "mu", "rest"):
            arrs = []
            for c in calls:
                a = c[key]
                arrs.append(np.concatenate([a, np.zeros((C - a.shape[0],) + a.shape[1:], dtype=a.dtype)]))
            blob["%s_call_%s" % (name, key)] = np.stack(arrs)
        print(name, "contacts per step (world 0):", res[0][2].tolist(), "final t",
              [round(float(r[3][-1]), 4) for r in res], "engine calls", len(calls))
    path = os.path.join(OUT, "bworld_joints.npz")
    np.savez_compressed(path, **blob)
    print("->", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
