"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference's `World.step_dt` for circles among static convex
polygon obstacles, in the REFERENCE's formulation: every obstacle is a body with 3 dofs pinned by a
`TotalConstraint` (constraints.py:176-192), listed after the circles, exactly as a reference `World` built from
`[Circle..., Rect / Hull...]` with one `TotalConstraint` per obstacle.

Extends `oracle.world_oracle.OracleCircleWorld` with the circle-hull contact of contacts.py:84-144 (the closest point
of the polygon when the centre is outside -- the reference reaches it by GJK --, the max-separation edge (SAT) when
the centre is inside). The GPU side (`BatchedWorld(obstacles=...)`) eliminates the pinned dofs instead (one-body
contacts); the two formulations cross-check each other. PARITY PIN: tests/test_obstacle_oracle.py against
trajectories recorded from the unmodified reference (tests/golden/bworld_obstacles.npz).
"""
import torch

from .world_oracle import OracleCircleWorld


def _rot(a):
    c, s = torch.cos(a), torch.sin(a)
    return torch.stack([torch.stack([c, -s]), torch.stack([s, c])])


def hull_centroid(verts):
    """bodies.py:216-226."""
    num, den = 0, 0
    for i in range(len(verts)):
        v1, v2 = verts[i], verts[(i + 1) % len(verts)]
        cross = v2[0] * v1[1] - v2[1] * v1[0]
        num = num + cross * (v1 + v2)
        den = den + cross / 2
    return num / (6 * den)


def hull_inertia(verts, mass):
    """bodies.py:179-189 (vertices about the centroid)."""
    num, den = 0, 0
    for i in range(len(verts)):
        v1, v2 = verts[i], verts[(i + 1) % len(verts)]
        nc = abs(v2[0] * v1[1] - v2[1] * v1[0])
        num = num + nc * (v1 @ v1 + v1 @ v2 + v2 @ v2)
        den = den + nc
    return mass * num / den / 6


def circle_polygon(c, verts):
    """contacts.py:84-144 for one circle centre c [2] and world-frame vertices [V, 2]: returns ('out', q) with q the
    closest point, or ('in', n, sep) with the outward normal and separation of the max-separation edge."""
    V = verts.shape[0]
    area = sum(verts[e, 0] * verts[(e + 1) % V, 1] - verts[e, 1] * verts[(e + 1) % V, 0] for e in range(V))
    orient = 1.0 if area > 0 else -1.0
    best_q, best_d2, best_sep, best_n = None, float("inf"), -float("inf"), None
    inside = True
    for e in range(V):
        a, b = verts[e], verts[(e + 1) % V]
        ed = b - a
        if not ed.norm().item() > 0:                         # a repeated vertex: no edge
            continue
        n = orient * torch.stack([ed[1], -ed[0]]) / ed.norm()
        sp = n @ (c - a)
        if sp.item() > 0:
            inside = False
        if sp.item() > best_sep:
            best_sep, best_n = sp.item(), (n, sp)
        t = ((c - a) @ ed / (ed @ ed)).clamp(0.0, 1.0)
        q = a + t * ed
        d2 = ((c - q) ** 2).sum()
        if d2.item() < best_d2:
            best_d2, best_q = d2.item(), q
    if inside:
        return ("in",) + best_n
    return ("out", best_q)


class OracleObstacleWorld(OracleCircleWorld):
    """Circles (pos [nc,2], rad, vel [nc,3], mass, restitution, fric_coeff) plus static convex polygons
    `obstacles` (list of world-frame vertex tensors [V, 2]) with masses / friction / restitution, all pinned.
    `obstacle_rot`: the bodies' initial rotation p[0] (a `Rect((rot, x, y), dims)` starts at rot; only the
    recorded state depends on it, the vertices are the world-frame ones given)."""

    def __init__(self, pos, rad, vel, mass, restitution, fric_coeff, obstacles, obstacle_fric=0.9,
                 obstacle_rest=0.5, obstacle_mass=1.0, obstacle_rot=0.0, gravity=100.0, dt=1.0 / 30, eps=0.1, tol=1e-6,
                 post_stab=False, max_iter=10):
        f64 = torch.float64
        pos = torch.as_tensor(pos, dtype=f64)
        ncirc, no = pos.shape[0], len(obstacles)
        as_list = lambda x: [float(x)] * no if not hasattr(x, "__len__") else [float(t) for t in x]
        self.ncirc, self.no = ncirc, no
        self.local, cents, inert = [], [], []
        om, orot = as_list(obstacle_mass), as_list(obstacle_rot)
        for k, v in enumerate(obstacles):
            v = torch.as_tensor(v, dtype=f64)
            cen = hull_centroid(v)
            # Hull.verts: about the centroid (bodies.py:170-173), stored at rotation 0
            self.local.append((v - cen) @ _rot(torch.tensor(orot[k], dtype=f64)))
            cents.append(cen)
            inert.append(hull_inertia(v - cen, om[k]))
        rad_c = torch.as_tensor(rad, dtype=f64).reshape(-1)
        super().__init__(torch.cat([pos, torch.stack(cents)]) if no else pos,
                         torch.cat([rad_c, torch.ones(no, dtype=f64)]),
                         torch.cat([torch.as_tensor(vel, dtype=f64).reshape(ncirc, 3), torch.zeros(no, 3, dtype=f64)]),
                         torch.cat([torch.as_tensor(mass, dtype=f64).reshape(-1), torch.tensor(om, dtype=f64)]),
                         torch.cat([torch.as_tensor(restitution, dtype=f64).reshape(-1),
                                    torch.tensor(as_list(obstacle_rest), dtype=f64)]),
                         torch.cat([torch.as_tensor(fric_coeff, dtype=f64).reshape(-1),
                                    torch.tensor(as_list(obstacle_fric), dtype=f64)]),
                         gravity=gravity, static=list(range(ncirc, ncirc + no)), dt=dt, eps=eps, tol=tol,
                         post_stab=post_stab, max_iter=max_iter)
        for k in range(no):                                  # Hull / Rect inertia (bodies.py:179-189, :269-270)
            self.Md[3 * (ncirc + k)] = inert[k]
            self.p[ncirc + k, 0] = orot[k]
        self.find_contacts()

    def obstacle_verts(self, k):
        b = self.ncirc + k
        return self.p[b, 1:] + self.local[k] @ _rot(self.p[b, 0]).t()

    def find_contacts(self):
        cs = []
        nc = self.ncirc
        verts = [self.obstacle_verts(k) for k in range(self.no)] if hasattr(self, "local") else []
        for i in range(nc):
            for j in range(i + 1, nc + len(verts)):
                c = self.p[i, 1:]
                if j < nc:
                    nrm = c - self.p[j, 1:]
                    dist = nrm.norm()
                    pen = self.rad[i] + self.rad[j] - dist
                    if pen.item() < -self.eps:
                        continue
                    nrm = nrm / dist
                    cs.append((nrm, -nrm * (self.rad[i] - pen / 2), nrm * (self.rad[j] - pen / 2), pen, i, j))
                    continue
                hit = circle_polygon(c, verts[j - nc])
                if hit[0] == "out":
                    q = hit[1]
                    best_dist = (q - c).norm() - self.rad[i]
                    if best_dist.item() > self.eps:
                        continue
                    nrm = (c - q) / (c - q).norm()
                else:
                    nrm, sp = hit[1], hit[2]
                    best_dist = sp - self.rad[i]
                    q = c - nrm * sp
                cs.append((nrm, q - c, q - self.p[j, 1:], -best_dist, i, j))
        self.contacts = cs
