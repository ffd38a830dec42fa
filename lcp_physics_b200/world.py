"""`BatchedWorld`: B independent 2-D worlds of circles stepped in lock-step on one GPU (SURVEY.md f-1).

The reference steps ONE scene per `World` object on the host (physics/world.py:72-122) and calls the
LCP with batch = 1 (SURVEY.md F3); `run_world` already anticipates a list of worlds (world.py:250-252).
Here the state of B scenes lives in structure-of-arrays tensors on the GPU and one step is

    new_v           <- -LCP(contact list)            lcpb200_engine_forward, mode 0   (engines.py:50-76)
    p               <- p + new_v dt_s                bodies.py:80-96, per-scene dt halving on penetration
                                                      (world.py:88-107)
    dp              <- -LCP_poststab(contact list)/2 lcpb200_engine_forward, mode 1   (engines.py:80-116,
                                                      world.py:109-120), optional

with contact generation for circle pairs (contacts.py:68-80: normal = (pos1 - pos2)/dist, penetration =
r1 + r2 - dist, contact when penetration >= -eps, p1 = -n (r1 - pen/2), p2 = n (r2 - pen/2)) on the device:
the pair test and the ordered compaction of all nb (nb - 1) / 2 pairs by lcpb200_find_contacts
(csrc/lcp_contacts.cuh), pair order (i < j, lexicographic) as the reference's broadphase callback visits
them, the geometry of the selected pairs by torch ops (differentiable). Every scene keeps its OWN contact count: the fused kernels take a per-scene count, and a scene
without contacts gets the equality-constrained solve of engines.py:35-49 inside the same kernel.

Scope (what the reference's demos use that this class mirrors): `Circle` bodies (bodies.py:114-140),
`Gravity` (forces.py), `TotalConstraint` pins (constraints.py:176-192), restitution / friction as the
mean of the two bodies (world.py:144-151, :213-224), `eps`, `tol`, `post_stab`, `strict_no_penetration`.
Hulls (`Rect`, `Hull`), joints between bodies and the renderer are not mirrored (SURVEY.md section 8f).
Everything is differentiable through torch autograd (the LCP through lcpb200_engine_backward). Scenes of up to
42 bodies (3 nb + 3 n_static <= 128) use the condensed-KKT kernels (fp32 / fp64); larger scenes (BASELINE
config 4: a 512-ball pile) the banded large-scene kernels (csrc/lcp_banded.cuh), float64.
"""
import ctypes

import torch

from . import _lib
from .engines import engine_solve


class BatchedWorld:
    def __init__(self, pos, rad, vel=None, mass=1.0, restitution=0.5, fric_coeff=0.9, gravity=10.0,
                 static=(), gravity_mask=None, dt=1.0 / 30, eps=0.1, tol=1e-6, post_stab=False,
                 strict_no_penetration=True, max_iter=10, contact_capacity=None, device=None, exact_adjoint=False):
        """pos [B,nb,2], rad [B,nb] (or [nb] / scalar), vel [B,nb,3] (rot, x, y) or None, mass / restitution /
        fric_coeff [B,nb] (or broadcastable), `static`: indices of bodies pinned by a TotalConstraint,
        `gravity`: g of the `Gravity` force (forces.py) applied to the bodies in gravity_mask
        (default: every non-static body). `exact_adjoint`: backward() through every LCP solve uses the true
        adjoint (the transposed KKT system, DESIGN.md section 3.4); the default False reproduces the reference's
        gradients, which are biased for every step with friction. Forward results do not depend on it."""
        _lib.require_cuda()
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        pos = torch.as_tensor(pos)
        self.dtype = pos.dtype if pos.dtype in (torch.float32, torch.float64) else torch.float64
        to = lambda t: torch.as_tensor(t, dtype=self.dtype).to(self.device)
        pos = to(pos)
        B, nb, _ = pos.shape
        self.B, self.nb, self.n = B, nb, 3 * nb
        bc = lambda t: to(t).expand(B, nb).contiguous() if torch.as_tensor(t).dim() < 2 else to(t)
        self.rad, self.mass = bc(rad), bc(mass)
        self.restitution, self.fric_coeff = bc(restitution), bc(fric_coeff)
        self.inertia = self.mass * self.rad * self.rad / 2                          # bodies.py:126
        self.p = torch.cat([pos.new_zeros(B, nb, 1), pos], 2)                       # (rot, x, y)  bodies.py:27-33
        self.v = to(vel).reshape(B, self.n).clone() if vel is not None else pos.new_zeros(B, self.n)
        self.static = [int(k) for k in static]
        gm = torch.ones(nb, dtype=torch.bool)
        gm[self.static] = False
        if gravity_mask is not None:
            gm = torch.as_tensor(gravity_mask, dtype=torch.bool)
        self.fext = pos.new_zeros(B, self.n)
        if gravity is not None:
            self.fext[:, 2::3] = self.mass * float(gravity) * gm.to(self.device).to(self.dtype)   # Gravity: DOWN * m * g
        self.ne = 3 * len(self.static)
        if self.ne:
            A = pos.new_zeros(self.ne, self.n)
            for r, k in enumerate(self.static):
                for q in range(3):
                    A[3 * r + q, 3 * k + q] = 1.0                                  # TotalConstraint.J = eye(3)
            self.A = A.unsqueeze(0).expand(B, -1, -1).contiguous()
        else:
            self.A = None
        self.dt, self.eps, self.tol = float(dt), float(eps), float(tol)
        self.post_stab, self.strict_no_pen, self.max_iter = post_stab, strict_no_penetration, max_iter
        self.exact_adjoint = bool(exact_adjoint)
        ii, jj = torch.triu_indices(nb, nb, 1)
        self.pi, self.pj = ii.to(self.device), jj.to(self.device)                   # pair (i, j), i < j, lexicographic
        self.cap = int(contact_capacity) if contact_capacity else min(int(self.pi.numel()), 3 * nb)
        # 3 nb + 3 n_static <= 128 and <= 256 contacts: condensed-KKT kernels (fp32 / fp64, differentiable);
        # larger scenes: the banded large-scene kernels (fp64; lcp_banded.cuh)
        self.large = self.n + self.ne > 128 or 4 * self.cap > 1024
        if self.large and (self.dtype != torch.float64 or self.ne > 16):
            raise ValueError("BatchedWorld: scenes with 3 nb + 3 n_static > 128 (or > 256 contacts) need float64 "
                             "and at most 5 pinned bodies")
        self.t = pos.new_zeros(B)
        self.find_contacts()
        if self.strict_no_pen and bool((self.max_penetration() > self.tol).any()):
            raise AssertionError("Interpenetration at start")                      # world.py:66-68

    # ------------------------------------------------------------------ contacts.py:68-80, batched
    def find_contacts(self):
        """Pair test + ordered compaction on the GPU (lcpb200_find_contacts: all nb (nb - 1) / 2 pairs of every
        scene, lexicographic order = the reference's contact order), then the contact geometry of the selected
        pairs with torch ops (differentiable w.r.t. the positions)."""
        lib = _lib.load()
        B, cap, dev = self.B, self.cap, self.device
        pos = self.p[:, :, 1:]
        pos_c = pos.detach().contiguous()
        b1 = torch.empty(B, cap, dtype=torch.int32, device=dev)
        b2 = torch.empty(B, cap, dtype=torch.int32, device=dev)
        counts = torch.empty(B, dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(lib.lcpb200_find_contacts(_lib.dtype_code(self.dtype), B, self.nb, cap, self.eps, _lib.ptr(pos_c),
                                                 _lib.ptr(self.rad), _lib.ptr(b1), _lib.ptr(b2), _lib.ptr(counts),
                                                 ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
        if int(counts.max()) > cap:
            raise RuntimeError("BatchedWorld: a scene has %d contacts, capacity %d" % (int(counts.max()), cap))
        self.c_b1, self.c_b2, self.counts = b1, b2, counts
        needs_graph = torch.is_grad_enabled() and any(t.requires_grad for t in (self.p, self.rad, self.fric_coeff, self.restitution))
        if not needs_graph:
            # nothing to differentiate: the geometry of the selected pairs in one kernel as well
            new = lambda *s_: torch.empty(B, cap, *s_, dtype=self.dtype, device=dev)
            self.c_normal, self.c_p1, self.c_p2 = new(2), new(2), new(2)
            self.c_pen, self.c_mu, self.c_rest = new(), new(), new()
            with torch.cuda.device(dev):
                _lib.check(lib.lcpb200_contact_geometry(
                    _lib.dtype_code(self.dtype), B, self.nb, cap, _lib.ptr(pos_c), _lib.ptr(self.rad.detach().contiguous()),
                    _lib.ptr(self.fric_coeff.detach().contiguous()), _lib.ptr(self.restitution.detach().contiguous()),
                    _lib.ptr(b1), _lib.ptr(b2), _lib.ptr(counts),
                    *[_lib.ptr(t) for t in (self.c_normal, self.c_p1, self.c_p2, self.c_pen, self.c_mu, self.c_rest)],
                    ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
            return
        i1, i2 = b1.long(), b2.long()
        take = lambda t, idx: torch.gather(t, 1, idx)
        d = torch.gather(pos, 1, i1.unsqueeze(2).expand(-1, -1, 2)) - torch.gather(pos, 1, i2.unsqueeze(2).expand(-1, -1, 2))
        dist = d.norm(dim=2)                                                       # b1.pos - b2.pos   contacts.py:69-71
        r1, r2 = take(self.rad, i1), take(self.rad, i2)
        pen_c = r1 + r2 - dist
        normal = d / dist.unsqueeze(2)
        valid = torch.arange(cap, device=dev).unsqueeze(0) < counts.unsqueeze(1)
        self.c_normal = normal
        self.c_p1 = -normal * (r1 - pen_c / 2).unsqueeze(2)                        # contacts.py:75-77
        self.c_p2 = normal * (r2 - pen_c / 2).unsqueeze(2)
        self.c_pen = torch.where(valid, pen_c, pen_c.new_full((), -1e30))
        self.c_b1, self.c_b2 = b1, b2
        self.c_mu = 0.5 * (take(self.fric_coeff, i1) + take(self.fric_coeff, i2))              # world.py:213-224
        self.c_rest = 0.5 * (take(self.restitution, i1) + take(self.restitution, i2))          # world.py:144-151
        self.counts = counts

    def find_contacts_torch(self):
        """The same contact list with torch ops only (O(nb^2) tensors, a stable sort for the compaction): the
        independent implementation tests/test_gpu_world.py checks lcpb200_find_contacts against. Returns
        (counts, b1, b2)."""
        pos = self.p[:, :, 1:]
        d = pos[:, self.pi] - pos[:, self.pj]
        pen = self.rad[:, self.pi] + self.rad[:, self.pj] - d.norm(dim=2)
        active = pen >= -self.eps                                                  # `if penetration < -eps: return`
        counts = active.sum(1)
        order = torch.sort((~active).to(torch.int8), dim=1, stable=True)[1][:, :self.cap]   # active pairs first, in pair order
        return counts.to(torch.int32), self.pi[order].to(torch.int32), self.pj[order].to(torch.int32)

    def max_penetration(self):
        return self.c_pen.max(dim=1)[0]

    # ------------------------------------------------------------------ engine calls
    def _lcp(self, mode, dt, b):
        z, status = engine_solve(self.mass, self.inertia, self.v, self.fext, self.c_normal, self.c_p1, self.c_p2,
                                 self.c_mu, self.c_rest, self.c_b1, self.c_b2, dt, A=self.A, b=b, mode=mode,
                                 max_iter=self.max_iter if mode == 0 else 10, exact_adjoint=self.exact_adjoint,
                                 counts=self.counts)
        if bool((status == _lib.STATUS_SINGULAR_Q).any()):
            from .lcp import SINGULAR_Q_MSG
            raise RuntimeError(SINGULAR_Q_MSG)
        if bool((status == -100).any()):
            raise RuntimeError("BatchedWorld: a scene's contact topology is not supported by the fused kernel")
        return z

    def solve_dynamics(self, dt):
        """engines.py:26-78 for every scene: new_v = -zhat."""
        b = self.v.new_zeros(self.B, self.ne) if self.ne else None
        return -self._lcp(0, dt, b)

    def post_stabilization(self):
        """engines.py:80-116 for every scene: -zhat with b = Je v."""
        b = torch.bmm(self.A, self.v.unsqueeze(2)).squeeze(2) if self.ne else None
        return -self._lcp(1, 0.0, b)

    # ------------------------------------------------------------------ world.py:72-122
    def step(self):
        self.step_dt(self.dt)

    def step_dt(self, dt):
        start_p = self.p.clone()
        self.v = self.solve_dynamics(dt)
        dts = self.v.new_full((self.B,), float(dt))
        done = torch.zeros(self.B, dtype=torch.bool, device=self.device)
        while True:
            moved = start_p + self.v.reshape(self.B, self.nb, 3) * dts.reshape(self.B, 1, 1)      # body.move(dt)
            self.p = torch.where(done.reshape(self.B, 1, 1), self.p, moved)
            self.find_contacts()
            ok = self.max_penetration() <= self.tol
            if not self.strict_no_pen:
                ok = ok | (dts < self.dt / 4)                                      # world.py:98-100
            done = done | ok
            if bool(done.all()):
                break
            dts = torch.where(done, dts, dts / 2)                                  # world.py:101 (positions reset: start_p)
        if self.post_stab:
            tmp_v = self.v
            dp = self.post_stabilization() / 2                                     # world.py:111-112
            self.p = self.p + dp.reshape(self.B, self.nb, 3) * dts.reshape(self.B, 1, 1)
            self.v = tmp_v
            self.find_contacts()
        self.t = self.t + dts

    def get_v(self):
        return self.v

    def get_p(self):
        return self.p.reshape(self.B, self.n)
