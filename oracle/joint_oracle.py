"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference's `World.step_dt` with CONSTRAINTS between bodies,
pairs excluded from contact and time-dependent external forces, for circles, dynamic `Rect` / `Hull` bodies and pinned
obstacles (oracle/polygon_oracle.py).

Extends `oracle.polygon_oracle.OracleHullWorld` with
  * the reference's constraint objects (constraints.py:13-173) restated on body indices: `J()`, `move`, `update_pos`,
    including the Joint's polar bookkeeping (r1, rot1 from cart_to_polar; rot1 advanced by v_rot(body1) dt at every
    move, pos1 = polar_to_cart(r1, rot1)) and the reset of rot1 to its start value when dt is halved (world.py:85,
    :104-107);
  * `Je()` (world.py:156-170): the pinned obstacles' TotalConstraint rows first, then the constraints in list order
    (the order tests/golden/make_joint_world_golden.py hands them to the reference World);
  * the `no_contact` skip of the contact handler (contacts.py:60, Body.add_no_contact);
  * a force function of t added to gravity (ExternalForce, forces.py), evaluated once per step at world.t
    (engines.py:27-32), with gravity on the bodies of `gravity_mask` only.
PARITY PIN: tests/test_joint_oracle.py against trajectories recorded from the unmodified reference
(tests/golden/bworld_joints.npz).
"""
import math

import torch

from .polygon_oracle import OracleHullWorld

f64 = torch.float64


def cart_to_polar(v):
    """utils.py:75-82 (positive=True)."""
    r = v.norm()
    theta = torch.atan2(v[1], v[0])
    if theta.item() < 0:
        theta = theta + 2 * math.pi
    return r, theta


def polar_to_cart(r, theta):
    """utils.py:85-90."""
    return torch.cat([torch.cos(theta).unsqueeze(0), torch.sin(theta).unsqueeze(0)]).squeeze() * r


class Joint:
    """constraints.py:13-53 between bodies i and j (None: the world point pos). rot2 is advanced by the reference but
    never read by J(), so it is not kept."""
    num_constraints = 2

    def __init__(self, world, i, j, pos):
        self.w, self.i, self.j = world, i, j
        self.pos = torch.as_tensor(pos, dtype=f64).clone()
        self.pos1 = self.pos - self.w.p[i, 1:]
        self.r1, self.rot1 = cart_to_polar(self.pos1)
        if j is not None:
            self.pos2 = self.pos - self.w.p[j, 1:]

    def J(self):
        J1 = torch.stack([torch.stack([-self.pos1[1], torch.tensor(1.0, dtype=f64), torch.tensor(0.0, dtype=f64)]),
                          torch.stack([self.pos1[0], torch.tensor(0.0, dtype=f64), torch.tensor(1.0, dtype=f64)])])
        J2 = None
        if self.j is not None:
            J2 = torch.stack([torch.stack([self.pos2[1], torch.tensor(-1.0, dtype=f64), torch.tensor(0.0, dtype=f64)]),
                              torch.stack([-self.pos2[0], torch.tensor(0.0, dtype=f64),
                                           torch.tensor(-1.0, dtype=f64)])])
        return J1, J2

    def move(self, dt, v):
        self.rot1 = self.rot1 + v[3 * self.i] * dt
        self.update_pos()

    def update_pos(self):
        self.pos1 = polar_to_cart(self.r1, self.rot1)
        self.pos = self.w.p[self.i, 1:] + self.pos1
        if self.j is not None:
            self.pos2 = self.pos - self.w.p[self.j, 1:]


class FixedJoint:
    """constraints.py:56-92."""
    num_constraints = 3

    def __init__(self, world, i, j):
        self.w, self.i, self.j = world, i, j
        self.rot1 = torch.tensor(0.0, dtype=f64)
        self.update_pos()

    def J(self):
        J1 = torch.zeros(3, 3, dtype=f64)
        J1[0, 0], J1[1, 0] = -self.pos1[1], self.pos1[0]
        J1[0, 1] = J1[1, 2] = J1[2, 0] = 1.0
        J2 = torch.zeros(3, 3, dtype=f64)
        J2[0, 0], J2[1, 0] = self.pos2[1], -self.pos2[0]
        J2[0, 1] = J2[1, 2] = J2[2, 0] = -1.0
        return J1, J2

    def move(self, dt, v):
        self.update_pos()

    def update_pos(self):
        self.pos = self.w.p[self.i, 1:]
        self.pos1 = self.pos - self.w.p[self.i, 1:]
        self.pos2 = self.pos - self.w.p[self.j, 1:]


class AxisConstraint:
    """XConstraint (dof 1), YConstraint (dof 2), RotConstraint (dof 0): constraints.py:95-173."""
    num_constraints = 1

    def __init__(self, world, i, dof):
        self.w, self.i, self.j, self.dof = world, i, None, dof
        self.rot1 = self.w.p[i, 0]

    def J(self):
        J = torch.zeros(1, 3, dtype=f64)
        J[0, self.dof] = 1.0
        return J, None

    def move(self, dt, v):
        self.update_pos()

    def update_pos(self):
        self.rot1 = self.w.p[self.i, 0]


class OracleJointWorld(OracleHullWorld):
    """OracleHullWorld plus `constraints` (list of ("joint", i, j, anchor) / ("fixed", i, j) / ("x" | "y" | "rot", i),
    body indices in [circles, polygons]), `no_contact` (pairs of indices in [circles, polygons, obstacles]),
    `gravity_mask` (bools over the dynamic bodies; default all) and `force` (f(t) -> [ndyn, 3] (rot, x, y), added to
    gravity)."""

    def __init__(self, *args, constraints=(), no_contact=(), gravity_mask=None, force=None, **kw):
        self.no_contact = {(min(a, b), max(a, b)) for a, b in no_contact}
        super().__init__(*args, **kw)
        self.force = force
        if gravity_mask is not None:
            for k, on in enumerate(gravity_mask):
                if not on:
                    self.f[3 * k + 2] = 0.0
        self.f_gravity = self.f.clone()
        self.Je_static = self.Je.clone()
        axis = {"x": 1, "y": 2, "rot": 0}
        self.cons = []
        for c in constraints:
            if c[0] == "joint":
                self.cons.append(Joint(self, c[1], c[2], c[3]))
            elif c[0] == "fixed":
                self.cons.append(FixedJoint(self, c[1], c[2]))
            else:
                self.cons.append(AxisConstraint(self, c[1], axis[c[0]]))
        self.Je = self.Je_()

    def Je_(self):
        """world.py:156-170."""
        rows = sum(c.num_constraints for c in self.cons)
        Je = torch.zeros(rows, self.n, dtype=f64)
        r = 0
        for c in self.cons:
            J1, J2 = c.J()
            Je[r:r + J1.shape[0], 3 * c.i:3 * c.i + 3] = J1
            if J2 is not None:
                Je[r:r + J2.shape[0], 3 * c.j:3 * c.j + 3] = J2
            r += J1.shape[0]
        return torch.cat([self.Je_static, Je])

    def apply_forces(self, t):
        if self.force is None:
            return self.f_gravity
        ext = torch.zeros(self.n, dtype=f64)
        ext[:3 * self.ndyn] = torch.as_tensor(self.force(t), dtype=f64).reshape(-1)
        return self.f_gravity + ext

    def find_contacts(self):
        super().find_contacts()
        if getattr(self, "no_contact", None):
            self.contacts = [c for c in self.contacts if (c[4], c[5]) not in self.no_contact]   # contacts.py:60

    def step(self):
        """world.py:83-122 with joints: moved after the bodies, rot1 reset on dt halving, moved by the
        post-stabilisation's dp."""
        dt = self.dt
        start_p = self.p.clone()
        start_rot = [c.rot1 for c in self.cons]
        self.Je = self.Je_()
        self.f = self.apply_forces(self.t)
        self.v = self.solve_dynamics(dt)
        while True:
            self._set_p(start_p + self.v.reshape(self.nb, 3) * dt)
            for c in self.cons:
                c.move(dt, self.v)
            self.find_contacts()
            if all(c[3].item() <= self.tol for c in self.contacts):
                break
            dt /= 2
            self._set_p(start_p.clone())
            for c, r in zip(self.cons, start_rot):
                c.rot1 = r.clone()
                c.update_pos()
        if self.post_stab:
            self.Je = self.Je_()
            dp = self.post_stabilization() / 2
            self._set_p(self.p + dp.reshape(self.nb, 3) * dt)
            for c in self.cons:
                c.move(dt, dp)
            self.find_contacts()
        self.t += dt
