"""Records trajectories of B independent UNMODIFIED reference `World`s (ode/pygame stubbed, oracle/ref_shim.py) of
circles falling into a bin of static `Rect`s, for `BatchedWorld(obstacles=...)` and oracle/obstacle_oracle.py to
reproduce:

    python tests/golden/make_obstacle_world_golden.py        (build container only)

Scene: a `Rect` floor, two `Rect` walls and one tilted `Rect` ramp, each pinned by a `TotalConstraint` and listed
AFTER the circles (the order BatchedWorld's pair walk follows); the obstacles do not touch each other, so the
reference adds no hull-hull rows. Six circles (radius 15, Gravity g = 100): two on the ramp, three just above the
floor, one against the right wall, with per-scene jitter, velocities, masses, friction and restitution.
`random` is seeded (the reference seeds its circle-hull GJK with random.choice).
Stored per variant (post_stab off / on): p, v of every body, the contact count and t after every step; and the
contact list the first step solves with (normal, p1, p2, penetration, body1, body2 per scene).
"""
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
from lcp_physics.physics.constraints import TotalConstraint  # noqa: E402
from lcp_physics.physics.forces import Gravity  # noqa: E402
from lcp_physics.physics.world import World  # noqa: E402

ref_engines.LCPFunction = ref_shim.ReferenceLCPFunction
OUT = os.path.dirname(os.path.abspath(__file__))
B, STEPS, RAD = 3, 30, 15.0
# (rot, x, y), dims, friction, restitution: floor, left wall, right wall, ramp
OBSTACLES = [((0.0, 300.0, 520.0), (400.0, 20.0), 0.8, 0.4),
             ((0.0, 85.0, 400.0), (20.0, 200.0), 0.5, 0.5),
             ((0.0, 515.0, 400.0), (20.0, 200.0), 0.5, 0.5),
             ((0.3, 200.0, 380.0), (120.0, 10.0), 0.6, 0.3)]


def _on_ramp(dx, gap):
    a, (cx, cy) = OBSTACLES[3][0][0], OBSTACLES[3][0][1:]
    c, s = np.cos(a), np.sin(a)
    return (cx + c * dx + 5.0 * s + (RAD + gap) * s, cy + s * dx - 5.0 * c - (RAD + gap) * c)


# centres (x, y) and the gap to the surface below (resting within eps = 0.1: contacts from the first step on)
CIRCLES = [(_on_ramp(-15.0, 0.0), 0.03), (_on_ramp(25.0, 0.0), 0.06), ((330.0, 495.0), 0.02), ((362.0, 495.0), 0.05),
           ((346.0, 462.0), 1.5), ((490.0 - 0.04, 470.0), 0.0)]


def initial(seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda: float(torch.rand(1, generator=g))
    pos = []
    for (x, y), gap in CIRCLES:
        a = 0.02 * r()
        if x > 480:                                  # against the right wall: move along it, keep the gap
            pos.append([x, y - 3.0 * r()])
        elif y > 490:                                # on the floor
            pos.append([x + 0.6 * r(), y - gap - a])
        elif y > 440:                                # above the two floor balls
            pos.append([x + 0.6 * r(), y - gap])
        else:                                        # on the ramp (its normal is (sin 0.3, -cos 0.3))
            pos.append([x + (gap + a) * np.sin(0.3), y - (gap + a) * np.cos(0.3)])
    vel = [[0.1 * (r() - 0.5), 4.0 * (r() - 0.5), 4.0 * (r() - 0.5)] for _ in CIRCLES]
    mass = [0.5 + r() for _ in CIRCLES]
    fric = [0.2 + 0.7 * r() for _ in CIRCLES]
    rest = [0.2 + 0.5 * r() for _ in CIRCLES]
    return dict(pos=np.array(pos), vel=np.array(vel), mass=np.array(mass), fric=np.array(fric), rest=np.array(rest),
                rad=np.full(len(CIRCLES), RAD))


def build(ic, post_stab):
    bodies, joints = [], []
    for k in range(len(CIRCLES)):
        c = Circle(list(ic["pos"][k]), RAD, vel=tuple(ic["vel"][k]), mass=float(ic["mass"][k]),
                   restitution=float(ic["rest"][k]), fric_coeff=float(ic["fric"][k]))
        c.add_force(Gravity(g=100))
        bodies.append(c)
    for pos, dims, fr, re in OBSTACLES:
        o = Rect(list(pos), list(dims), restitution=re, fric_coeff=fr)
        joints.append(TotalConstraint(o))
        bodies.append(o)
    return World(bodies, joints, dt=1.0 / 30, post_stab=post_stab)


def run(ic, post_stab):
    world = build(ic, post_stab)
    cs = world.contacts
    first = dict(normal=np.array([c[0][0].detach().numpy() for c in cs]), p1=np.array([c[0][1].detach().numpy() for c in cs]),
                 p2=np.array([c[0][2].detach().numpy() for c in cs]),
                 pen=np.array([float(c[0][3]) for c in cs]), b1=np.array([c[1] for c in cs]), b2=np.array([c[2] for c in cs]))
    P, V, NC, T = [], [], [], []
    for _ in range(STEPS):
        world.step()
        P.append(torch.stack([b.p for b in world.bodies]).detach().numpy().copy())
        V.append(world.v.detach().numpy().reshape(-1, 3).copy())
        NC.append(len(world.contacts))
        T.append(float(world.t))
    return np.stack(P), np.stack(V), np.array(NC), np.array(T), first


def main():
    random.seed(0)
    torch.manual_seed(0)
    ics = [initial(200 + k) for k in range(B)]
    blob = {k: np.stack([ic[k] for ic in ics]) for k in ics[0]}
    w0 = build(ics[0], False)
    blob["obst_verts"] = np.stack([(torch.stack(o.verts) + o.pos).detach().numpy() for o in w0.bodies[len(CIRCLES):]])
    blob["obst_pos"] = np.array([o[0] for o in OBSTACLES])
    blob["obst_dims"] = np.array([o[1] for o in OBSTACLES])
    blob["obst_fric"] = np.array([o[2] for o in OBSTACLES])
    blob["obst_rest"] = np.array([o[3] for o in OBSTACLES])
    for tag, ps in (("nops", False), ("ps", True)):
        res = [run(ic, ps) for ic in ics]
        blob[tag + "_p"] = np.stack([r[0] for r in res], 1)          # [steps, B, nb + no, 3]
        blob[tag + "_v"] = np.stack([r[1] for r in res], 1)
        blob[tag + "_nc"] = np.stack([r[2] for r in res], 1)
        blob[tag + "_t"] = np.stack([r[3] for r in res], 1)
        if not ps:
            C = max(len(r[4]["pen"]) for r in res)
            for key in ("normal", "p1", "p2", "pen", "b1", "b2"):
                arrs = []
                for r in res:
                    a = r[4][key]
                    pad = np.zeros((C - a.shape[0],) + a.shape[1:], dtype=a.dtype)
                    arrs.append(np.concatenate([a.reshape((-1,) + a.shape[1:]), pad]))
                blob["first_" + key] = np.stack(arrs)
            blob["first_n"] = np.array([len(r[4]["pen"]) for r in res])
        print(tag, "contacts per step (world 0):", res[0][2].tolist(), "final t", [round(float(r[3][-1]), 4) for r in res])
    path = os.path.join(OUT, "bworld_obstacles.npz")
    np.savez_compressed(path, **blob)
    print("->", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
