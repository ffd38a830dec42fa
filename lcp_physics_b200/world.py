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
mean of the two bodies (world.py:144-151, :213-224), `eps`, `tol`, `post_stab`, `strict_no_penetration`,
and STATIC convex polygon obstacles -- the reference's `Rect` / `Hull` floors, walls and ramps pinned by a
`TotalConstraint` (`obstacles=`, `rect_vertices`): a pinned body has zero velocity, so its equality rows are
eliminated exactly and a contact against it is a one-body contact (body2 >= nb, include/lcpb200.h) whose rows touch
only the circle's three columns (DESIGN.md section 9), and DYNAMIC convex polygons -- the reference's `Rect` / `Hull`
bodies (`polygons=`), ordered after the circles and before the obstacles, with the hull-hull contact rule of
contacts.py:145-292 (SAT + reference-face clipping, 0-2 contacts per pair) detected by lcpb200_body_contacts. Joints
between bodies and the renderer are not mirrored (SURVEY.md section 8f).
Everything is differentiable through torch autograd (the LCP through lcpb200_engine_backward). Scenes of up to
42 dynamic bodies (3 (nb + npoly) + 3 n_static <= 128) use the condensed-KKT kernels (fp32 / fp64); larger scenes
(BASELINE config 4: a 512-ball pile) the banded large-scene kernels (csrc/lcp_banded.cuh), float64.
"""
import ctypes
import math

import torch

from . import _lib
from .engines import engine_solve


def rect_vertices(pos, dims, angle=0.0):
    """World-frame vertices [4, 2] of the reference's `Rect(pos, dims)` rotated by `angle` (bodies.py:253-290: half
    dims v0 = (w/2, h/2), v1 = (-w/2, h/2), vertices [v0, v1, -v0, -v1] about the centre, rotated by
    [[cos, -sin], [sin, cos]]). Differentiable in every argument (tensors or numbers)."""
    ref = next((t for t in (pos, dims, angle) if isinstance(t, torch.Tensor)), None)
    dt_ = ref.dtype if ref is not None and ref.is_floating_point() else torch.float64
    dev = ref.device if ref is not None else None
    pos, dims, angle = [torch.as_tensor(t, dtype=dt_, device=dev) for t in (pos, dims, angle)]
    h = dims / 2
    v0, v1 = h, h * h.new_tensor([-1.0, 1.0])
    local = torch.stack([v0, v1, -v0, -v1])
    c, s = torch.cos(angle), torch.sin(angle)
    rot = torch.stack([torch.stack([c, -s]), torch.stack([s, c])])
    return pos + local @ rot.t()


def polygon_centroid(verts):
    """Area centroid [..., 2] of polygons [..., V, 2] (bodies.py:216-226: the reference point of a `Hull`)."""
    a, b = verts, torch.roll(verts, -1, dims=-2)
    cross = b[..., 0] * a[..., 1] - b[..., 1] * a[..., 0]
    return (cross.unsqueeze(-1) * (a + b)).sum(-2) / (6 * (cross.sum(-1) / 2).unsqueeze(-1))


def check_obstacles(verts, B, name="obstacles"):
    """Validates obstacle vertices [no, V, 2] (shared by the batch) or [B, no, V, 2]; returns them as [B, no, V, 2].
    Every polygon must have >= 3 vertices, a non-zero area and be convex (the contact rule of contacts.py:84-144 is
    the one for convex hulls). All polygons share V: a polygon with fewer vertices may repeat one (its zero-length
    edges are skipped by the contact rule). `name` labels the error messages."""
    v = torch.as_tensor(verts)
    if v.dim() == 3:
        v = v.unsqueeze(0).expand(B, -1, -1, -1)
    if v.dim() != 4 or v.shape[0] != B or v.shape[3] != 2:
        raise ValueError("%s: need vertices [n, V, 2] or [B, n, V, 2] (B = %d), got %s" % (name, B, tuple(v.shape)))
    if v.shape[1] == 0:
        raise ValueError("%s: no polygon given (pass %s=None)" % (name, name))
    if v.shape[2] < 3:
        raise ValueError("%s: every polygon needs at least 3 vertices" % name)
    if v.shape[2] > 256:
        raise ValueError("%s: at most 256 vertices per polygon" % name)
    w = v.detach().double()
    if not bool(torch.isfinite(w).all()):
        raise ValueError("%s: non-finite vertex" % name)
    e = torch.roll(w, -1, dims=2) - w
    deg = ~(e.norm(dim=-1) > 0)                          # zero-length edges: a vertex repeated to pad to the common V
    en, found = torch.roll(e, -1, dims=2), ~torch.roll(deg, -1, dims=2)
    for s_ in range(2, v.shape[2]):                      # the next edge of non-zero length
        ok = ~found & ~torch.roll(deg, -s_, dims=2)
        en = torch.where(ok.unsqueeze(-1), torch.roll(e, -s_, dims=2), en)
        found = found | ok
    # cross product of consecutive edges; collinear vertices (|turn| at round-off level) are allowed
    turn = (e[..., 0] * en[..., 1] - e[..., 1] * en[..., 0]) / (e.norm(dim=-1) * en.norm(dim=-1)).clamp_min(1e-300)
    turn = torch.where(deg, torch.zeros_like(turn), turn)
    area = (w[..., 0] * torch.roll(w, -1, dims=2)[..., 1] - w[..., 1] * torch.roll(w, -1, dims=2)[..., 0]).sum(-1)
    if bool((area.abs() <= 0).any()):
        raise ValueError("%s: a polygon has zero area" % name)
    tol = math.sqrt(torch.finfo(v.dtype).eps) if v.is_floating_point() else 1e-8    # coordinates rounded to v.dtype
    if bool(((turn * area.sign().unsqueeze(-1)) < -tol).any()):
        raise ValueError("%s: every polygon must be convex" % name)
    return v


def check_polygons(verts, B):
    """Validates the vertices of dynamic polygons as check_obstacles does, and their orientation: a `Hull` asserts a
    positive shoelace area (bodies.py:169, :228-235, `_is_clockwise` in screen coordinates), which makes
    left_orthogonal(edge) the outward normal the hull-hull rule uses. Returns [B, npoly, V, 2]."""
    v = check_obstacles(verts, B, name="polygons")
    w = v.detach().double()
    area = (w[..., 0] * torch.roll(w, -1, dims=2)[..., 1] - w[..., 1] * torch.roll(w, -1, dims=2)[..., 0]).sum(-1)
    if bool((area < 0).any()):
        raise ValueError("polygons: vertices must be in the orientation of positive shoelace area (as Hull asserts); "
                         "reverse their order")
    return v


def polygon_inertia(rel, mass):
    """Hull's angular inertia (bodies.py:179-189) of polygons with vertices rel [..., V, 2] about their centroid:
    m / 6 * sum |v2 x v1| (v1.v1 + v1.v2 + v2.v2) / sum |v2 x v1|; for a rectangle it equals Rect's m (w^2 + h^2) / 12."""
    a, b = rel, torch.roll(rel, -1, dims=-2)
    nc = (b[..., 0] * a[..., 1] - b[..., 1] * a[..., 0]).abs()
    num = (nc * ((a * a).sum(-1) + (a * b).sum(-1) + (b * b).sum(-1))).sum(-1)
    return mass * num / nc.sum(-1) / 6


def _pad_vertices(v, V):
    """[B, n, V0, 2] -> [B, n, V, 2] (V >= V0) by repeating the last vertex: a zero-length edge, skipped by every rule."""
    if v.shape[2] == V:
        return v
    return torch.cat([v, v[:, :, -1:].expand(-1, -1, V - v.shape[2], -1)], 2)


class BatchedWorld:
    def __init__(self, pos, rad, vel=None, mass=1.0, restitution=0.5, fric_coeff=0.9, gravity=10.0,
                 static=(), gravity_mask=None, dt=1.0 / 30, eps=0.1, tol=1e-6, post_stab=False,
                 strict_no_penetration=True, max_iter=10, contact_capacity=None, device=None, exact_adjoint=False,
                 obstacles=None, obstacle_fric=0.9, obstacle_rest=0.5, polygons=None, poly_rot=0.0, poly_vel=None,
                 poly_mass=1.0, poly_fric=0.9, poly_rest=0.5):
        """pos [B,nb,2] (nb may be 0), rad [B,nb] (or [nb] / scalar), vel [B,nb,3] (rot, x, y) or None, mass /
        restitution / fric_coeff [B,nb] (or broadcastable).
        `polygons`: dynamic convex polygons, the reference's `Rect` / `Hull` bodies (bodies.py:154-301): world-frame
        vertices at the initial pose, [npoly, V, 2] (shared by the batch) or [B, npoly, V, 2], in the orientation of
        positive shoelace area (e.g. `rect_vertices`); `poly_rot`: their initial rotation p[0] ([B, npoly] or
        broadcastable), `poly_vel` [B, npoly, 3] or None, `poly_mass` / `poly_fric` / `poly_rest` [B, npoly] or
        broadcastable; all may require grad. A polygon's position is its area centroid and its inertia Hull's.
        Bodies are ordered [circles (nb), polygons (npoly), obstacles]: p, v, get_p(), get_v(), mass, inertia, fext
        and the `static` / `gravity_mask` indices cover the nb + npoly dynamic bodies in that order.
        `static`: indices of bodies pinned by a TotalConstraint,
        `gravity`: g of the `Gravity` force (forces.py) applied to the bodies in gravity_mask
        (default: every non-static body). `exact_adjoint`: backward() through every LCP solve uses the true
        adjoint (the transposed KKT system, DESIGN.md section 3.4); the default False reproduces the reference's
        gradients, which are biased for every step with friction. Forward results do not depend on it.
        `obstacles`: world-frame vertices of static convex polygons, [no, V, 2] (shared by the batch) or
        [B, no, V, 2] (e.g. `rect_vertices`; a polygon with fewer than V vertices repeats one); they may require
        grad. They act as the reference's pinned `Rect` / `Hull` bodies listed AFTER the circles: contact order,
        rule and material are those of such a World.
        `obstacle_fric` / `obstacle_rest`: their friction / restitution, [B,no] or broadcastable."""
        _lib.require_cuda()
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        pos = torch.as_tensor(pos)
        self.dtype = pos.dtype if pos.dtype in (torch.float32, torch.float64) else torch.float64
        to = lambda t: torch.as_tensor(t, dtype=self.dtype).to(self.device)
        pos = to(pos)
        B, nb, _ = pos.shape
        self.np = 0
        if polygons is not None:
            pv = check_polygons(polygons, B).to(device=self.device, dtype=self.dtype)  # [B,np,V,2], keeps its graph
            self.np = int(pv.shape[1])
        nd = nb + self.np                                                           # dynamic bodies
        if nd == 0:
            raise ValueError("BatchedWorld: no circle and no polygon given")
        self.B, self.nb, self.nd, self.n = B, nb, nd, 3 * nd
        bc = lambda t: to(t).expand(B, nb).contiguous() if torch.as_tensor(t).dim() < 2 else to(t)
        self.rad, self.mass = bc(rad), bc(mass)
        self.restitution, self.fric_coeff = bc(restitution), bc(fric_coeff)
        self.inertia = self.mass * self.rad * self.rad / 2                          # bodies.py:126
        self.p = torch.cat([pos.new_zeros(B, nb, 1), pos], 2)                       # (rot, x, y)  bodies.py:27-33
        v0 = to(vel).reshape(B, 3 * nb).clone() if vel is not None else pos.new_zeros(B, 3 * nb)
        if self.np:
            bp = lambda t: to(t).expand(B, self.np).contiguous() if torch.as_tensor(t).dim() < 2 else to(t)
            pmass, rot = bp(poly_mass), bp(poly_rot)
            self.pfric, self.prest = bp(poly_fric), bp(poly_rest)
            cen = polygon_centroid(pv)                                              # Hull.pos (bodies.py:170-173)
            rel = pv - cen.unsqueeze(2)
            c, s = torch.cos(rot).unsqueeze(2), torch.sin(rot).unsqueeze(2)
            # Hull.verts at rotation 0: R(-rot) (verts - centroid); every step rotates them by p[0] (bodies.py:202-214)
            self.plocal = torch.stack([c * rel[..., 0] + s * rel[..., 1], -s * rel[..., 0] + c * rel[..., 1]], 3)
            self.mass = torch.cat([self.mass, pmass], 1)
            self.inertia = torch.cat([self.inertia, polygon_inertia(rel, pmass)], 1)
            self.p = torch.cat([self.p, torch.cat([rot.unsqueeze(2), cen], 2)], 1)
            pvel = to(poly_vel).reshape(B, 3 * self.np) if poly_vel is not None else pos.new_zeros(B, 3 * self.np)
            v0 = torch.cat([v0, pvel], 1)
        self.v = v0
        self.static = [int(k) for k in static]
        gm = torch.ones(nd, dtype=torch.bool)
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
        self.no, self.nv = 0, 0
        if obstacles is not None:
            ov = check_obstacles(obstacles, B)
            self.ov = ov.to(device=self.device, dtype=self.dtype)                  # [B,no,V,2], keeps its graph
            self.no, self.nv = int(ov.shape[1]), int(ov.shape[2])
            bo = lambda t: to(t).expand(B, self.no).contiguous() if torch.as_tensor(t).dim() < 2 else to(t)
            self.ofric, self.orest = bo(obstacle_fric), bo(obstacle_rest)
            self.oref = polygon_centroid(self.ov)                                   # Hull.pos (bodies.py:166-173)
        if self.np:
            self.nv = max(self.nv, int(pv.shape[2]))                                # one common V for both groups
            self.plocal = _pad_vertices(self.plocal, self.nv)
            if self.no:
                self.ov = _pad_vertices(self.ov, self.nv)
        nt = nd + self.no
        ii, jj = torch.triu_indices(nt, nt, 1)
        if self.no:
            keep = ii < nd                                                          # obstacles never pair up
            ii, jj = ii[keep], jj[keep]
        self.pi, self.pj = ii.to(self.device), jj.to(self.device)                   # pair (i, j), i < j, lexicographic
        if self.np:
            # a polygon-polygon or polygon-obstacle pair may give 2 contacts
            most = int(self.pi.numel()) + int((self.pi >= nb).sum())
            self.cap = int(contact_capacity) if contact_capacity else max(1, min(most, (4 if self.no else 3) * nb + 8 * self.np))
        else:
            self.cap = int(contact_capacity) if contact_capacity else min(int(self.pi.numel()), (4 if self.no else 3) * nb)
        # 3 (nb + npoly) + 3 n_static <= 128 and <= 256 contacts: condensed-KKT kernels (fp32 / fp64,
        # differentiable); larger scenes: the banded large-scene kernels (fp64; lcp_banded.cuh)
        self.large = self.n + self.ne > 128 or 4 * self.cap > 1024
        if self.large and (self.dtype != torch.float64 or self.ne > 16):
            raise ValueError("BatchedWorld: scenes with 3 (nb + npoly) + 3 n_static > 128 (or > 256 contacts) need "
                             "float64 and at most 5 pinned bodies (static obstacles do not count)")
        self.t = pos.new_zeros(B)
        self.find_contacts()
        if self.strict_no_pen and bool((self.max_penetration() > self.tol).any()):
            raise AssertionError("Interpenetration at start")                      # world.py:66-68

    # ------------------------------------------------------------------ contacts.py:68-80, batched
    def find_contacts(self):
        """Pair test + ordered compaction on the GPU (lcpb200_find_contacts: all nb (nb - 1) / 2 pairs of every
        scene, lexicographic order = the reference's contact order), then the contact geometry of the selected
        pairs with torch ops (differentiable w.r.t. the positions)."""
        if self.np:
            return self._find_contacts_bodies()
        if self.no:
            return self._find_contacts_obstacles()
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

    def _find_contacts_obstacles(self):
        """find_contacts for worlds with static obstacles: lcpb200_world_contacts walks circle-circle and
        circle-obstacle pairs in the order of a reference World with bodies [circles..., obstacles...]; the geometry
        comes from the same call, or from torch ops (_geometry_torch) when something needs autograd."""
        lib = _lib.load()
        B, cap, dev = self.B, self.cap, self.device
        pos_c = self.p[:, :, 1:].detach().contiguous()
        b1 = torch.empty(B, cap, dtype=torch.int32, device=dev)
        b2 = torch.empty(B, cap, dtype=torch.int32, device=dev)
        counts = torch.empty(B, dtype=torch.int32, device=dev)
        needs_graph = torch.is_grad_enabled() and any(
            t.requires_grad for t in (self.p, self.rad, self.fric_coeff, self.restitution, self.ov, self.ofric, self.orest))
        d = lambda t: t.detach().contiguous()
        geo = [None] * 6
        if not needs_graph:
            new = lambda *s_: torch.empty(B, cap, *s_, dtype=self.dtype, device=dev)
            geo = [new(2), new(2), new(2), new(), new(), new()]
        with torch.cuda.device(dev):
            _lib.check(lib.lcpb200_world_contacts(
                _lib.dtype_code(self.dtype), B, self.nb, self.no, self.nv, cap, self.eps, _lib.ptr(pos_c),
                *[_lib.ptr(d(t)) for t in (self.rad, self.fric_coeff, self.restitution, self.ov, self.oref, self.ofric,
                                           self.orest)],
                _lib.ptr(b1), _lib.ptr(b2), _lib.ptr(counts), *[_lib.ptr(t) for t in geo],
                ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
        if int(counts.max()) > cap:
            raise RuntimeError("BatchedWorld: a scene has %d contacts, capacity %d" % (int(counts.max()), cap))
        self.c_b1, self.c_b2, self.counts = b1, b2, counts
        if not needs_graph:
            self.c_normal, self.c_p1, self.c_p2, self.c_pen, self.c_mu, self.c_rest = geo
            return
        self.c_normal, self.c_p1, self.c_p2, pen, self.c_mu, self.c_rest = self._geometry_torch(b1, b2)
        valid = torch.arange(cap, device=dev).unsqueeze(0) < counts.unsqueeze(1)
        self.c_pen = torch.where(valid, pen, pen.new_full((), -1e30))

    def polygon_vertices(self):
        """World-frame vertices [B, npoly, V, 2] of the dynamic polygons at the current p: centroid + R(rot) local
        (Hull.set_p / rotate_verts, bodies.py:202-214), differentiable in p and the polygons' initial vertices."""
        q = self.p[:, self.nb:]
        c, s = torch.cos(q[:, :, 0:1]), torch.sin(q[:, :, 0:1])
        lx, ly = self.plocal[..., 0], self.plocal[..., 1]
        return torch.stack([q[:, :, 1:2] + (c * lx - s * ly), q[:, :, 2:3] + (s * lx + c * ly)], 3)

    def _find_contacts_bodies(self):
        """find_contacts for worlds with dynamic polygons: lcpb200_body_contacts walks the pairs of the body list
        [circles..., polygons..., obstacles...] (circle-circle, circle-polygon and hull-hull rules; 0-2 contacts per
        pair) and returns each hull-hull contact's features; the geometry comes from the same call, or from torch ops
        that rebuild it from those features (_geometry_torch) when something needs autograd."""
        lib = _lib.load()
        B, cap, dev, nb = self.B, self.cap, self.device, self.nb
        pverts = self.polygon_vertices()
        pcen = self.p[:, nb:, 1:]
        b1 = torch.empty(B, cap, dtype=torch.int32, device=dev)
        b2 = torch.empty(B, cap, dtype=torch.int32, device=dev)
        feat = torch.empty(B, cap, dtype=torch.int32, device=dev)
        counts = torch.empty(B, dtype=torch.int32, device=dev)
        obst = (self.ov, self.oref, self.ofric, self.orest) if self.no else (None,) * 4
        needs_graph = torch.is_grad_enabled() and any(
            t is not None and t.requires_grad
            for t in (self.p, self.rad, self.fric_coeff, self.restitution, self.plocal, self.pfric, self.prest) + obst)
        d = lambda t: t.detach().contiguous() if t is not None else None
        geo = [None] * 6
        if not needs_graph:
            new = lambda *s_: torch.empty(B, cap, *s_, dtype=self.dtype, device=dev)
            geo = [new(2), new(2), new(2), new(), new(), new()]
        # contiguous copies held until the call returns (a temporary's memory could be reused before the kernel runs)
        ins = [d(t) for t in (self.p[:, :nb, 1:], self.rad, self.fric_coeff, self.restitution, pverts, pcen, self.pfric,
                              self.prest) + obst]
        with torch.cuda.device(dev):
            _lib.check(lib.lcpb200_body_contacts(
                _lib.dtype_code(self.dtype), B, nb, self.np, self.no, self.nv, cap, self.eps, *[_lib.ptr(t) for t in ins],
                _lib.ptr(b1), _lib.ptr(b2), _lib.ptr(counts), _lib.ptr(feat), *[_lib.ptr(t) for t in geo],
                ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
        if int(counts.max()) > cap:
            raise RuntimeError("BatchedWorld: a scene has %d contacts, capacity %d" % (int(counts.max()), cap))
        self.c_b1, self.c_b2, self.c_feat, self.counts = b1, b2, feat, counts
        if not needs_graph:
            self.c_normal, self.c_p1, self.c_p2, self.c_pen, self.c_mu, self.c_rest = geo
            return
        self.c_normal, self.c_p1, self.c_p2, pen, self.c_mu, self.c_rest = self._geometry_torch(b1, b2, feat, pverts)
        valid = torch.arange(cap, device=dev).unsqueeze(0) < counts.unsqueeze(1)
        self.c_pen = torch.where(valid, pen, pen.new_full((), -1e30))

    def _hull_torch(self, i1, i2, feat, verts, ref):
        """Torch mirror of the hull-hull geometry of csrc/lcp_contacts.cuh (contacts.py:156-201, clip_segment_to_line
        :270-292) for the pairs (i1, i2) [B,C] of polygon bodies, REBUILT FROM THE KERNEL'S FEATURES feat [B,C] (which
        body holds the reference face, reference and incident edges, the first clip's outcome, which clipped point),
        so the graph path and the kernel path cannot select different features. verts [B,P,V,2] / ref [B,P,2]: the
        polygons [dynamic..., obstacles...] and their centroids. Returns normal, p1, p2, penetration."""
        nb, V = self.nb, self.nv
        P = verts.shape[1]
        f = feat.long().clamp_min(0)
        kind, clip1, ref2 = f & 3, (f >> 2) & 3, ((f >> 4) & 1).bool()
        re, ie = (f >> 5) & 255, (f >> 13) & 255
        k1, k2 = (i1 - nb).clamp(0, P - 1), (i2 - nb).clamp(0, P - 1)
        kr, ki = torch.where(ref2, k2, k1), torch.where(ref2, k1, k2)
        poly = lambda k: torch.gather(verts, 1, k.unsqueeze(2).unsqueeze(3).expand(-1, -1, V, 2))   # [B,C,V,2]
        Vr, Vi = poly(kr), poly(ki)
        take2 = lambda t, idx: torch.gather(t, 1, idx.unsqueeze(2).expand(-1, -1, 2))
        cr, ci = take2(ref, kr), take2(ref, ki)
        vtx = lambda Vx, e: torch.gather(Vx, 2, e.unsqueeze(2).unsqueeze(3).expand(-1, -1, 1, 2)).squeeze(2)
        Wr = torch.roll(Vr, -1, dims=2)
        area = (Vr[..., 0] * Wr[..., 1] - Vr[..., 1] * Wr[..., 0]).sum(2)
        orient = torch.where(area > 0, 1.0, -1.0).to(verts.dtype)
        E = vtx(Vr, (re + 1) % V) - vtx(Vr, re)
        ln = E.norm(dim=2)
        ln1 = torch.where(ln > 0, ln, torch.ones_like(ln))
        n = torch.stack([orient * E[..., 1] / ln1, -orient * E[..., 0] / ln1], 2)   # outward normal of the reference edge
        r = vtx(Vr, re) - cr
        h = (ln / 2).unsqueeze(2)
        v0, v1 = vtx(Vi, ie) - cr, vtx(Vi, (ie + 1) % V) - cr                        # incident edge, reference frame
        cp = torch.stack([n[..., 1], -n[..., 0]], 2)                                # clip plane left_orthogonal(n)
        dot = lambda a, b: (a * b).sum(2, keepdim=True)
        safe = lambda x: torch.where(x != 0, x, torch.ones_like(x))
        d0, d1 = dot(cp, v0) + h, dot(cp, v1) + h
        c1 = v0 + d0 / safe(d0 - d1) * (v1 - v0)
        a = torch.where((clip1 == 2).unsqueeze(2), v1, v0)
        b = torch.where((clip1 == 0).unsqueeze(2), v1, c1)
        e0, e1 = dot(-cp, a) + h, dot(-cp, b) + h
        c2 = a + e0 / safe(e0 - e1) * (b - a)
        k_ = kind.unsqueeze(2)
        v = torch.where(k_ == 0, v0, torch.where(k_ == 1, v1, torch.where(k_ == 2, c1, c2)))
        dist = dot(n, v - r)
        q = v + n * -dist                                                           # on the reference edge's line
        s = q + cr - ci
        w = ref2.unsqueeze(2)
        return torch.where(w, n, -n), torch.where(w, s, q), torch.where(w, q, s), -dist.squeeze(2)

    def _circle_polygon_torch(self, c, k, verts=None):
        """Torch mirror of csrc/lcp_contacts.cuh circle_polygon for circle centres c [B,P,2] against polygons
        k [B,P] (long) of verts (default: the obstacles): (inside, closest point q, squared distance, separating-edge
        normal, separation)."""
        B, P = k.shape
        verts = self.ov if verts is None else verts
        V = torch.gather(verts, 1, k.reshape(B, P, 1, 1).expand(B, P, self.nv, 2))          # [B,P,V,2]
        Wv = torch.roll(V, -1, dims=2)
        E = Wv - V
        area = (V[..., 0] * Wv[..., 1] - V[..., 1] * Wv[..., 0]).sum(2)
        orient = torch.where(area > 0, 1.0, -1.0).to(V.dtype).unsqueeze(2)
        ln = E.norm(dim=3)
        dg = ~(ln > 0)                                     # zero-length edges (repeated vertices): skipped, as the kernel
        ln1 = torch.where(dg, torch.ones_like(ln), ln)     # keeps the skipped entries finite, gradients too
        nrm = torch.stack([orient * E[..., 1] / ln1, -orient * E[..., 0] / ln1], 3)        # outward unit normals
        rel = c.unsqueeze(2) - V
        sp = torch.where(dg, torch.full_like(ln, -math.inf), (nrm * rel).sum(3))
        inside = ~(sp > 0).any(2)
        ee = (E * E).sum(3)
        t = ((rel * E).sum(3) / torch.where(dg, torch.ones_like(ee), ee)).clamp(0.0, 1.0)
        Q = V + t.unsqueeze(3) * E
        d2 = torch.where(dg, torch.full_like(ln, math.inf), ((c.unsqueeze(2) - Q) ** 2).sum(3))
        em = d2.argmin(2, keepdim=True)
        q = torch.gather(Q, 2, em.unsqueeze(3).expand(-1, -1, 1, 2)).squeeze(2)
        es = sp.argmax(2, keepdim=True)
        n_in = torch.gather(nrm, 2, es.unsqueeze(3).expand(-1, -1, 1, 2)).squeeze(2)
        sep = torch.gather(sp, 2, es).squeeze(2)
        return inside, q, torch.gather(d2, 2, em).squeeze(2), n_in, sep

    def _geometry_torch(self, b1, b2, feat=None, pverts=None):
        """Differentiable geometry and material of the selected pairs (circle-circle: contacts.py:69-77;
        circle-polygon: contacts.py:84-144, as lcpb200_world_contacts; hull-hull: _hull_torch, from the kernel's
        features feat), gradients reaching positions, radii, materials and the polygon / obstacle vertices.
        pverts: the dynamic polygons' world-frame vertices (worlds with polygons)."""
        nb = self.nb
        pos = self.p[:, :, 1:]
        i1, i2 = b1.long(), b2.long()
        take = lambda t, idx: torch.gather(t, 1, idx)
        take2 = lambda t, idx: torch.gather(t, 1, idx.unsqueeze(2).expand(-1, -1, 2))
        if self.np:                                  # polygon k of body nb + k: [dynamic polygons..., obstacles...]
            cat = lambda a, b: torch.cat([a, b], 1) if self.no else a
            polys, pref = cat(pverts, self.ov if self.no else None), cat(pos[:, nb:], self.oref if self.no else None)
            pfr = cat(self.pfric, self.ofric if self.no else None)
            prs = cat(self.prest, self.orest if self.no else None)
            hh = i1 >= nb
            n_h, p1_h, p2_h, pen_h = self._hull_torch(i1, i2, feat, polys, pref)
            kh1 = (i1 - nb).clamp_min(0)
            mu_h = 0.5 * (take(pfr, kh1) + take(pfr, (i2 - nb).clamp_min(0)))
            rest_h = 0.5 * (take(prs, kh1) + take(prs, (i2 - nb).clamp_min(0)))
            if nb == 0:
                return n_h, p1_h, p2_h, pen_h, mu_h, rest_h
            i1 = torch.where(hh, 0, i1)
        else:
            polys, pref, pfr, prs = self.ov, self.oref, self.ofric, self.orest
        cc = i2 < nb
        j = torch.where(cc, i2, 0)
        k = torch.where(cc, 0, i2 - nb)
        c = take2(pos, i1)
        r1 = take(self.rad, i1)
        one = torch.zeros_like(c)
        one[..., 0] = 1.0
        # circle-circle (slots of obstacle pairs get a harmless unit offset: no 0 / 0 in either pass)
        dcc = torch.where(cc.unsqueeze(2), c - take2(pos, j), one)
        dist = dcc.norm(dim=2)
        r2 = take(self.rad, j)
        pen_cc = r1 + r2 - dist
        n_cc = dcc / dist.unsqueeze(2)
        p1_cc = -n_cc * (r1 - pen_cc / 2).unsqueeze(2)
        p2_cc = n_cc * (r2 - pen_cc / 2).unsqueeze(2)
        # circle-obstacle / circle-polygon
        inside, q, _, n_in, sep = self._circle_polygon_torch(c, k, polys)
        out = ~cc & ~inside
        dq = torch.where(out.unsqueeze(2), c - q, one)
        dq_n = dq.norm(dim=2)
        n_co = torch.where(inside.unsqueeze(2), n_in, dq / dq_n.unsqueeze(2))
        pen_co = torch.where(inside, r1 - sep, r1 - dq_n)
        q_co = torch.where(inside.unsqueeze(2), c - n_in * sep.unsqueeze(2), q)   # best_pt2 = center - n (dist + rad)
        p1_co = q_co - c
        p2_co = q_co - take2(pref, k)
        w = cc.unsqueeze(2)
        normal = torch.where(w, n_cc, n_co)
        p1 = torch.where(w, p1_cc, p1_co)
        p2 = torch.where(w, p2_cc, p2_co)
        pen = torch.where(cc, pen_cc, pen_co)
        f1, e1 = take(self.fric_coeff, i1), take(self.restitution, i1)
        mu = 0.5 * (f1 + torch.where(cc, take(self.fric_coeff, j), take(pfr, k)))          # world.py:213-224
        rest = 0.5 * (e1 + torch.where(cc, take(self.restitution, j), take(prs, k)))       # world.py:144-151
        if self.np:
            h = hh.unsqueeze(2)
            return (torch.where(h, n_h, normal), torch.where(h, p1_h, p1), torch.where(h, p2_h, p2),
                    torch.where(hh, pen_h, pen), torch.where(hh, mu_h, mu), torch.where(hh, rest_h, rest))
        return normal, p1, p2, pen, mu, rest

    def find_contacts_torch(self):
        """The same contact list with torch ops only (O(nb^2) tensors, a stable sort for the compaction): the
        independent implementation tests/test_gpu_world.py checks lcpb200_find_contacts against (and
        tests/test_gpu_obstacles.py lcpb200_world_contacts). Returns (counts, b1, b2). Not available for worlds with
        dynamic polygons: their hull-hull rule is checked against the CPU oracle (oracle/polygon_oracle.py)."""
        if self.np:
            raise NotImplementedError("find_contacts_torch: worlds with dynamic polygons (see oracle/polygon_oracle.py)")
        pos = self.p[:, :, 1:]
        if self.no:
            nb = self.nb
            cc = self.pj < nb
            B = self.B
            pj = torch.where(cc, self.pj, 0)
            d = pos[:, self.pi] - pos[:, pj]
            pen = self.rad[:, self.pi] + self.rad[:, pj] - d.norm(dim=2)
            k = torch.where(cc, 0, self.pj - nb).unsqueeze(0).expand(B, -1)
            inside, _, d2, _, _ = self._circle_polygon_torch(pos[:, self.pi], k)
            hit_o = inside | ~(d2.sqrt() - self.rad[:, self.pi] > self.eps)              # contacts.py:110-112
            active = torch.where(cc, pen >= -self.eps, hit_o)
            counts = active.sum(1)
            order = torch.sort((~active).to(torch.int8), dim=1, stable=True)[1][:, :self.cap]
            return counts.to(torch.int32), self.pi[order].to(torch.int32), self.pj[order].to(torch.int32)
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
            moved = start_p + self.v.reshape(self.B, self.nd, 3) * dts.reshape(self.B, 1, 1)      # body.move(dt)
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
            self.p = self.p + dp.reshape(self.B, self.nd, 3) * dts.reshape(self.B, 1, 1)
            self.v = tmp_v
            self.find_contacts()
        self.t = self.t + dts

    def get_v(self):
        return self.v

    def get_p(self):
        return self.p.reshape(self.B, self.n)
