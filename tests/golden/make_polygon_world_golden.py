"""Records trajectories of B independent UNMODIFIED reference `World`s (ode/pygame stubbed, oracle/ref_shim.py) with
DYNAMIC `Rect` / `Hull` bodies, for `BatchedWorld(polygons=...)` and oracle/polygon_oracle.py to reproduce:

    python tests/golden/make_polygon_world_golden.py        (build container only)

Bodies are listed [circles..., dynamic Rect / Hull..., pinned Rect...] (the order BatchedWorld's pair walk follows),
every obstacle pinned by a `TotalConstraint`, Gravity g = 100 on every dynamic body. Two scenes, B worlds each with
per-world jitter of positions, rotations, velocities and materials:
  * slide: slide_demo's Rect (60 x 60, demos/demo.py:93-114) released just above a pinned Rect ramp tilted by pi / 32
    and slightly rotated against it, so it lands on a corner (1-point manifold) and then slides on a face (2 points);
  * stack: a pinned floor between two walls holding three Rects stacked, a tilted Rect falling onto a corner, a
    non-symmetric Hull (pentagon) standing on an edge with a small Rect on its top edge near one end (the clip window
    about the pentagon's centroid is off-centre), and three circles: one on the top box, one on the floor against the
    bottom box, one on the floor against that circle.
No box starts exactly parallel to its support: equal separations of two edges would be settled by rounding (the
reference's SAT scan order), so every recorded contact has a unique winning separation.
`random` is seeded (the reference seeds its circle-hull GJK with random.choice).
Stored per scene and variant (post_stab off / on): p, v of every body, the contact count and t after every step; the
contact list the first step solves with; and the initial bodies as the reference holds them (Hull.verts about the
centroid, p, mass, M[0, 0], materials, which are Rects).
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
from lcp_physics.physics.bodies import Circle, Hull, Rect  # noqa: E402
from lcp_physics.physics.constraints import TotalConstraint  # noqa: E402
from lcp_physics.physics.forces import Gravity  # noqa: E402
from lcp_physics.physics.world import World  # noqa: E402

ref_engines.LCPFunction = ref_shim.ReferenceLCPFunction
OUT = os.path.dirname(os.path.abspath(__file__))
B = 3
STEPS = {"slide": 40, "stack": 30}
PENTAGON = [[25.0, 0.0], [15.0, 30.0], [-15.0, 15.0], [-30.0, -15.0], [0.0, -30.0]]   # tests/test_hull.py, halved


def _rot(a, v):
    c, s = math.cos(a), math.sin(a)
    return np.array([c * v[0] - s * v[1], s * v[0] + c * v[1]])


def rect_bottom(cx, cy, w, h, a):
    """world-frame bottom corners (local (+-w/2, h/2); y grows downwards) of a Rect at (cx, cy) rotated by a"""
    return [np.array([cx, cy]) + _rot(a, (sx * w / 2, h / 2)) for sx in (-1, 1)]


def top_line(cx, cy, w, h, a):
    """y(x) of the line through the top edge of a Rect"""
    mid = np.array([cx, cy]) + _rot(a, (0.0, -h / 2))
    return lambda x: mid[1] + (x - mid[0]) * math.tan(a)


def place_on(line, cx, w, h, a, gap):
    """centre y of a Rect at x = cx rotated by a whose lowest bottom corner is `gap` above `line`"""
    lo = max(c[1] - line(c[0]) for c in rect_bottom(cx, 0.0, w, h, a))
    return -lo - gap


def slide_scene(seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda: float(torch.rand(1, generator=g))
    incl = math.pi / 32
    ramp = ((incl, 500.0, 300.0), (900.0, 10.0))
    a = incl + 0.01 + 0.02 * r()
    cx = 150.0 + 40.0 * r()
    cy = place_on(top_line(500.0, 300.0, 900.0, 10.0, incl), cx, 60.0, 60.0, a, 0.02 + 0.05 * r())
    rects = [((a, cx, cy), (60.0, 60.0), [0.5 * (r() - 0.5), 4.0 * (r() - 0.5), 4.0 * (r() - 0.5)], 1.0 + r(),
              0.15 + 0.3 * r(), 0.2 + 0.5 * r())]
    return dict(circles=[], rects=rects, hulls=[], obstacles=[ramp + (0.15, 0.5)])


def stack_scene(seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda: float(torch.rand(1, generator=g))
    jit = lambda: 0.004 * (r() - 0.5) + 0.002
    floor = ((0.0, 300.0, 520.0), (400.0, 20.0))
    obst = [floor + (0.8, 0.4), ((0.0, 85.0, 400.0), (20.0, 200.0), 0.5, 0.5),
            ((0.0, 515.0, 400.0), (20.0, 200.0), 0.5, 0.5)]
    fl = top_line(300.0, 520.0, 400.0, 20.0, 0.0)
    vel = lambda: [0.05 * (r() - 0.5), 2.0 * (r() - 0.5), 2.0 * (r() - 0.5)]
    mat = lambda: (0.5 + r(), 0.3 + 0.6 * r(), 0.2 + 0.4 * r())               # mass, friction, restitution
    rects = []
    x0 = 170.0 + 4.0 * r()
    below = fl
    for w, h in ((60.0, 30.0), (44.0, 26.0), (30.0, 20.0)):                   # the stack
        a = jit()
        cx = x0 + 2.0 * (r() - 0.5)
        cy = place_on(below, cx, w, h, a, 0.01 + 0.04 * r())
        rects.append(((a, cx, cy), (w, h), vel()) + mat())
        below = top_line(cx, cy, w, h, a)
    a = 0.35 + 0.05 * r()                                                       # the tilted Rect, on a corner
    cx = 250.0 + 4.0 * r()
    rects.append(((a, cx, place_on(fl, cx, 30.0, 30.0, a, 0.03 + 0.04 * r())), (30.0, 30.0), vel()) + mat())
    # the pentagon on its edge 3 -> 4 (rotated so that edge runs in -x: its outward normal points down), a small Rect
    # near one end of its upper edge of most upward normal
    pv = [np.array(v) for v in PENTAGON]
    e = pv[4] - pv[3]
    ap = math.pi - math.atan2(e[1], e[0]) + 0.003 + 0.002 * r()
    wv = [_rot(ap, v) for v in pv]
    px = 380.0 + 4.0 * r()
    py = fl(px) - max(v[1] for v in wv) - (0.01 + 0.04 * r())
    hull = ([[px + v[0], py + v[1]] for v in wv], vel()) + mat()
    up = lambda k: (wv[(k + 1) % 5] - wv[k])[0] / np.linalg.norm(wv[(k + 1) % 5] - wv[k])
    top = max(range(5), key=up)
    t0, t1 = wv[top] + np.array([px, py]), wv[(top + 1) % 5] + np.array([px, py])
    ta = math.atan2(t1[1] - t0[1], t1[0] - t0[0]) + 0.004 + 0.002 * r()
    tx = t0[0] + 0.7 * (t1[0] - t0[0])
    tl = lambda x: t0[1] + (x - t0[0]) * (t1[1] - t0[1]) / (t1[0] - t0[0])
    rects.append(((ta, tx, place_on(tl, tx, 16.0, 12.0, ta, 0.01 + 0.03 * r())), (16.0, 12.0), vel()) + mat())
    # circles (radius 10): on the top box, on the floor left of the bottom box, on the floor left of that circle
    (a2, c2x, c2y), (w2, h2) = rects[2][0], rects[2][1]
    x1 = c2x + 3.0 + 0.5 * (r() - 0.5)
    y1 = top_line(c2x, c2y, w2, h2, a2)(x1) - 10.0 / math.cos(a2) - (0.02 + 0.03 * r())
    (a0, c0x, c0y), (w0, h0) = rects[0][0], rects[0][1]
    left = min((np.array([c0x, c0y]) + _rot(a0, (-w0 / 2, sy * h0 / 2)))[0] for sy in (-1, 1))
    x2 = left - 10.0 - 0.08
    x3 = x2 - 20.0 - (0.02 + 0.05 * r())
    circles = [([x1, y1], vel()) + mat()]
    for x in (x2, x3):
        circles.append(([x, fl(x) - 10.0 - (0.01 + 0.04 * r())], vel()) + mat())
    return dict(circles=circles, rects=rects, hulls=[hull], obstacles=obst)


def build(sc, post_stab):
    bodies, joints = [], []
    for pos, vel, m, f, e in sc["circles"]:
        c = Circle(list(pos), 10.0, vel=tuple(vel), mass=m, fric_coeff=f, restitution=e)
        c.add_force(Gravity(g=100))
        bodies.append(c)
    for k, (pos, dims, vel, m, f, e) in enumerate(sc["rects"]):
        if k == len(sc["rects"]) - 1 and sc["hulls"]:
            for verts, hv, hm, hf, he in sc["hulls"]:                          # the pentagon before its top Rect
                h = Hull([0.0, 0.0], verts, vel=tuple(hv), mass=hm, fric_coeff=hf, restitution=he)
                h.add_force(Gravity(g=100))
                bodies.append(h)
        o = Rect(list(pos), list(dims), vel=tuple(vel), mass=m, fric_coeff=f, restitution=e)
        o.add_force(Gravity(g=100))
        bodies.append(o)
    for pos, dims, f, e in sc["obstacles"]:
        o = Rect(list(pos), list(dims), fric_coeff=f, restitution=e)
        joints.append(TotalConstraint(o))
        bodies.append(o)
    return World(bodies, joints, dt=1.0 / 30, post_stab=post_stab)


def run(sc, post_stab, steps):
    world = build(sc, post_stab)
    nc = len(sc["circles"])
    hs = world.bodies[nc:]
    V = max(len(b.verts) for b in hs)
    pad = lambda vs: np.stack([torch.stack(list(vs) + [vs[-1]] * (V - len(vs))).detach().numpy()])[0]
    init = dict(hull_verts=np.stack([pad(b.verts) for b in hs]), hull_nv=np.array([len(b.verts) for b in hs]),
                hull_p=np.stack([b.p.detach().numpy() for b in hs]), hull_vel=np.stack([b.v.detach().numpy() for b in hs]),
                hull_mass=np.array([float(b.mass) for b in hs]), hull_inertia=np.array([float(b.M[0, 0]) for b in hs]),
                hull_fric=np.array([float(b.fric_coeff) for b in hs]),
                hull_rest=np.array([float(b.restitution) for b in hs]),
                hull_is_rect=np.array([isinstance(b, Rect) for b in hs]),
                pos=np.array([b.pos.detach().numpy() for b in world.bodies[:nc]]).reshape(nc, 2),
                vel=np.array([b.v.detach().numpy() for b in world.bodies[:nc]]).reshape(nc, 3),
                mass=np.array([float(b.mass) for b in world.bodies[:nc]]),
                fric=np.array([float(b.fric_coeff) for b in world.bodies[:nc]]),
                rest=np.array([float(b.restitution) for b in world.bodies[:nc]]), rad=np.full(nc, 10.0))
    cs = world.contacts
    first = dict(normal=np.array([c[0][0].detach().numpy() for c in cs]).reshape(-1, 2),
                 p1=np.array([c[0][1].detach().numpy() for c in cs]).reshape(-1, 2),
                 p2=np.array([c[0][2].detach().numpy() for c in cs]).reshape(-1, 2),
                 pen=np.array([float(c[0][3]) for c in cs]), b1=np.array([c[1] for c in cs], dtype=np.int64),
                 b2=np.array([c[2] for c in cs], dtype=np.int64))
    P, Vv, NC, T = [], [], [], []
    for _ in range(steps):
        world.step()
        P.append(torch.stack([b.p for b in world.bodies]).detach().numpy().copy())
        Vv.append(world.v.detach().numpy().reshape(-1, 3).copy())
        NC.append(len(world.contacts))
        T.append(float(world.t))
    return np.stack(P), np.stack(Vv), np.array(NC), np.array(T), first, init


def main():
    random.seed(0)
    torch.manual_seed(0)
    blob = {}
    for name, make in (("slide", slide_scene), ("stack", stack_scene)):
        scenes = [make(300 + 17 * k + (0 if name == "slide" else 1000)) for k in range(B)]
        blob[name + "_nstatic"] = np.array(len(scenes[0]["obstacles"]))
        for tag, ps in (("nops", False), ("ps", True)):
            res = [run(sc, ps, STEPS[name]) for sc in scenes]
            pre = "%s_%s_" % (name, tag)
            blob[pre + "p"] = np.stack([r[0] for r in res], 1)           # [steps, B, nbodies, 3]
            blob[pre + "v"] = np.stack([r[1] for r in res], 1)
            blob[pre + "nc"] = np.stack([r[2] for r in res], 1)
            blob[pre + "t"] = np.stack([r[3] for r in res], 1)
            if not ps:
                for key in res[0][5]:
                    blob["%s_%s" % (name, key)] = np.stack([r[5][key] for r in res])
                C = max(len(r[4]["pen"]) for r in res)
                for key in ("normal", "p1", "p2", "pen", "b1", "b2"):
                    arrs = []
                    for r in res:
                        a = r[4][key]
                        pad = np.zeros((C - a.shape[0],) + a.shape[1:], dtype=a.dtype)
                        arrs.append(np.concatenate([a, pad]))
                    blob["%s_first_%s" % (name, key)] = np.stack(arrs)
                blob[name + "_first_n"] = np.array([len(r[4]["pen"]) for r in res])
            print(name, tag, "contacts per step (world 0):", res[0][2].tolist(),
                  "final t", [round(float(r[3][-1]), 4) for r in res])
    path = os.path.join(OUT, "bworld_polygons.npz")
    np.savez_compressed(path, **blob)
    print("->", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
