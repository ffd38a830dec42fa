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
the pair test and the ordered compaction of all nb (nb - 1) / 2 pairs by lcpb200_contacts
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
contacts.py:145-292 (SAT + reference-face clipping, 0-2 contacts per pair) detected by lcpb200_contacts, and
CONSTRAINTS between bodies (`constraints=`: `Joint`, `FixedJoint`, `XConstraint`, `YConstraint`, `RotConstraint`,
constraints.py:13-173) as equality rows of the engine's LCP, rebuilt with torch ops at every engine call, pairs excluded
from contact (`no_contact=`, Body.add_no_contact: skipped in the GPU pair walk of lcpb200_contacts) and
time-dependent external forces (`external_force=`, forces.py ExternalForce). The renderer is not mirrored.
Everything is differentiable through torch autograd (the LCP through lcpb200_engine_backward). Scenes of up to
42 dynamic bodies (3 (nb + npoly) + 3 n_static <= 128) use the condensed-KKT kernels (fp32 / fp64); larger scenes
(BASELINE config 4: a 512-ball pile) the banded large-scene kernels (csrc/lcp_banded.cuh), float64.
"""
import math

import numpy as np
import torch
import torch.autograd.forward_ad as fwAD

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


def _orientation(polys):
    """Orientation sign of polygons [..., V, 2] in their dtype: 1 where the shoelace area is positive
    (counter-clockwise), else -1 (poly_orient of csrc/lcp_contacts.cuh)."""
    W = torch.roll(polys, -1, dims=-2)
    area = (polys[..., 0] * W[..., 1] - polys[..., 1] * W[..., 0]).sum(-1)
    return torch.where(area > 0, 1.0, -1.0).to(polys.dtype)


def _edge_normal(E, orient, ln):
    """Outward unit normal orient (E_y, -E_x) / ln of edges E [..., 2] of polygons of orientation sign orient [...];
    ln is |E|, made non-zero by the caller where an edge is not used."""
    return torch.stack([orient * E[..., 1] / ln, -orient * E[..., 0] / ln], -1)


def _take2(t, idx):
    """Rows idx [B, n] of t [B, m, 2]: [B, n, 2]."""
    return torch.gather(t, 1, idx.unsqueeze(2).expand(-1, -1, 2))


def _polygons(pverts, ov):
    """The polygon bodies [B, P, V, 2] of a world, dynamic polygons then obstacles, from pverts (polygon_vertices())
    and ov (the obstacle vertices); either may be None, not both."""
    return torch.cat([t for t in (pverts, ov) if t is not None], 1)


def _detached(t):
    """t detached and contiguous, None for None: a kernel argument that stays alive until the call returns (a
    temporary's memory could be reused before the kernel runs)."""
    return t.detach().contiguous() if t is not None else None


def _chosen_edge(polys, body, edge, nb):
    """Edge `edge` of body `body` ([B, n] each) of a world whose polygons polys [B, P, V, 2] are bodies nb, nb + 1,
    ...: (v_e, v_f = the next vertex, E = v_f - v_e, the polygon's orientation sign [B, n]). Slots whose body is not a
    polygon read edge 0 of polygon 0, so that they stay finite."""
    B, _, V, _ = polys.shape
    is_p = body >= nb
    k = torch.where(is_p, body - nb, 0)
    e = torch.where(is_p, edge, 0)
    flat = polys.reshape(B, -1, 2)
    ve, vf = _take2(flat, k * V + e), _take2(flat, k * V + (e + 1) % V)
    return ve, vf, vf - ve, torch.gather(_orientation(polys), 1, k)


# ------------------------------------------------------------------ constraints.py:13-173, by body index
class Joint:
    """Revolute joint (constraints.py:13-53) between bodies i and j (j None: a joint to the world point `anchor`) at
    `anchor`, [2] (shared by the batch) or [B, 2], which may require grad. 2 equality rows."""
    num_constraints = 2

    def __init__(self, i, j, anchor):
        self.i, self.j, self.anchor = i, j, anchor

    def bodies(self):
        return (self.i,) if self.j is None else (self.i, self.j)


class FixedJoint:
    """Fixed joint (constraints.py:56-92): welds body j to body i. 3 equality rows."""
    num_constraints = 3

    def __init__(self, i, j):
        self.i, self.j = i, j

    def bodies(self):
        return (self.i, self.j)


class _AxisConstraint:
    num_constraints = 1
    dof = None                                    # the constrained coordinate of (rot, x, y)

    def __init__(self, i):
        self.i, self.j = i, None

    def bodies(self):
        return (self.i,)


class XConstraint(_AxisConstraint):
    """Prevents motion along x (constraints.py:122-146): the row [0, 1, 0] on body i."""
    dof = 1


class YConstraint(_AxisConstraint):
    """Prevents motion along y (constraints.py:95-119): the row [0, 0, 1] on body i."""
    dof = 2


class RotConstraint(_AxisConstraint):
    """Prevents rotation (constraints.py:149-173): the row [1, 0, 0] on body i."""
    dof = 0


def _cart_to_polar(v):
    """utils.py:75-82 (positive=True) per scene: r, theta of v [B, 2], theta in [0, 2 pi)."""
    r = v.norm(dim=1)
    th = torch.atan2(v[:, 1], v[:, 0])
    return r, torch.where(th < 0, th + 2 * math.pi, th)


def _polar_to_cart(r, th):
    """utils.py:85-90 per scene: [B, 2]."""
    return torch.stack([torch.cos(th) * r, torch.sin(th) * r], 1)


class _DetectFn(torch.autograd.Function):
    """Runs `fn(*tensors)`, a contact-detection kernel call, on plain tensors: under torch.func transforms (vjp in
    BatchedWorld.linearize) the arguments arrive unwrapped, so the kernel can read their storage. Its outputs --
    contact indices, counts, features and the kernel's geometry, which is used only when nothing is differentiated --
    are not differentiable."""

    @staticmethod
    def forward(fn, *tensors):
        return fn(*tensors)

    @staticmethod
    def setup_context(ctx, inputs, output):
        ctx.n_inputs = len(inputs)
        ctx.n_outputs = len(output)
        ctx.mark_non_differentiable(*output)

    @staticmethod
    def backward(ctx, *grads):
        return (None,) * ctx.n_inputs

    @staticmethod
    def jvp(ctx, *tangents):
        return (None,) * ctx.n_outputs

    @staticmethod
    def vmap(info, in_dims, fn, *tensors):
        # reached only when an argument is batched at this vmap level (jacfwd batches tangents, not the state)
        raise NotImplementedError("BatchedWorld: vmap over the world's state is not supported; batch scenes along "
                                  "dim 0 instead")


def _detect(fn, *tensors):
    """fn(*tensors); through _DetectFn when a torch.func transform has wrapped an argument (such a wrapper has no
    storage a kernel could read). Ordinary steps call the kernel directly."""
    if any(t is not None and torch._C._functorch.is_functorch_wrapped_tensor(t) for t in tensors):
        return _DetectFn.apply(fn, *tensors)
    return fn(*tensors)


def _has_tangent(t):
    """True when t carries a forward-mode tangent: an input of torch.func.jvp / jacfwd (a functorch-wrapped tensor) or
    a torch.autograd.forward_ad dual tensor. Forward mode leaves requires_grad False."""
    return t is not None and fwAD.unpack_dual(t).tangent is not None


def _needs_graph(tensors):
    """True when a result computed from `tensors` (None entries allowed) must be rebuilt with torch ops: one of them
    requires grad under grad mode, or carries a forward-mode tangent."""
    return (torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors)) or any(
        _has_tangent(t) for t in tensors)


def _max_dist(max_dist):
    """max_dist of a ray cast or signed distance as a float, finite and >= 0."""
    md = float(max_dist)
    if not math.isfinite(md) or md < 0:
        raise ValueError("max_dist: need a finite distance >= 0, got %r" % (max_dist,))
    return md


def _length(x, name):
    """A distance parameter (gap, skip, tol) as a float, finite and >= 0."""
    v = float(x)
    if not math.isfinite(v) or v < 0:
        raise ValueError("%s: need a finite value >= 0, got %r" % (name, x))
    return v


# default stop tolerance of time_of_impact / first_impact, in world units
TOI_TOL = {torch.float64: 1e-9, torch.float32: 1e-4}


def _check_count(v, name):
    """Rejects a count (rays, pixels) that is not an int >= 1; bool is not a count."""
    if isinstance(v, bool) or not isinstance(v, int) or v < 1:
        raise ValueError("%s: need an int >= 1, got %r" % (name, v))


MAX_ACTIVE_BODIES = 8192        # bodies of a world walked per scene (the kernel's shared-memory list of active bodies)


def check_active(active, B, nt):
    """Validates a per-scene activity mask, bool [B, nt] or broadcastable to it; returns it as a contiguous [B, nt]."""
    a = torch.as_tensor(active)
    if a.dtype != torch.bool:
        raise ValueError("active: need a bool mask [B, nb + npoly + no] = [%d, %d], got dtype %s" % (B, nt, a.dtype))
    try:
        a = a.expand(B, nt)
    except RuntimeError:
        raise ValueError("active: need a bool mask [B, nb + npoly + no] = [%d, %d] (or broadcastable), got %s"
                         % (B, nt, tuple(a.shape))) from None
    return a.contiguous()


def check_constraint_activity(cons, active):
    """A constraint takes part in scene s iff all its bodies are active there; raises ValueError, naming the scene and
    the constraint, when a constraint has both active and inactive bodies in some scene."""
    for ci, c in enumerate(cons):
        a = active[:, list(c.bodies())]
        mixed = (a.any(1) & ~a.all(1)).nonzero()
        if mixed.numel():
            raise ValueError("constraints: constraint %d (%s of bodies %s) has active and inactive bodies in scene %d; "
                             "a constraint takes part in a scene only with all its bodies active"
                             % (ci, type(c).__name__, c.bodies(), int(mixed[0, 0])))


def _no_contact_words(pairs, nt, where):
    """Bitmask [ceil(nt * nt / 32)] int32 of one pair list: bit i * nt + j (i < j) per excluded pair. Built from the
    pair list alone (nt * nt / 8 bytes: the layout the contact walk reads)."""
    prs = np.asarray([tuple(int(x) for x in pr) for pr in pairs], dtype=np.int64).reshape(-1, 2)
    bad = ~((prs >= 0) & (prs < nt)).all(1)
    if bad.any():
        raise ValueError("no_contact: body index out of range in %r%s (%d bodies)"
                         % (tuple(int(x) for x in prs[bad][0]), where, nt))
    same = prs[:, 0] == prs[:, 1]
    if same.any():
        a = int(prs[same][0, 0])
        raise ValueError("no_contact: the pair (%d, %d)%s names one body twice" % (a, a, where))
    bits = prs.min(1) * nt + prs.max(1)
    words = np.zeros((nt * nt + 31) // 32, dtype=np.uint32)
    np.bitwise_or.at(words, bits >> 5, (np.uint32(1) << (bits & 31).astype(np.uint32)))
    return torch.from_numpy(words.view(np.int32).copy())


def mask_bits(words, nt, i, j):
    """Bit i * nt + j of no_contact words ([W] or [B, W]) for the pairs (i, j) (long tensors, same device): True where
    the pair is excluded; [len(i)] or [B, len(i)]."""
    bit = i * nt + j
    return ((words[..., bit >> 5] >> (bit & 31).to(torch.int32)) & 1).bool()


def per_scene_pairs(pairs):
    """True when a `no_contact` argument is a list of pair lists, one per scene: its items are sequences of pairs,
    where a shared list's items are pairs of indices."""
    seq = lambda x: isinstance(x, (list, tuple))
    items = list(pairs)
    return bool(items) and all(seq(ps) and all(seq(pr) for pr in ps) for ps in items)


def no_contact_masks(pairs, B, nt):
    """The no_contact bitmask of lcpb200_contacts / lcpb200_contacts_active: for one pair list shared by the batch,
    words [ceil(nt * nt / 32)] int32; for a length-B list of pair lists (its items are sequences of pairs, where a
    shared list's items are pairs of indices), one row per scene, [B, ceil(nt * nt / 32)]: nt * nt / 8 bytes per
    scene (8 MB at the 8192-body bound), so per-scene lists suit worlds of up to a few hundred bodies."""
    items = list(pairs)
    if not per_scene_pairs(items):
        return _no_contact_words(items, nt, "")
    if len(items) != B:
        raise ValueError("no_contact: a per-scene list needs one pair list per scene (B = %d), got %d"
                         % (B, len(items)))
    return torch.stack([_no_contact_words(ps, nt, " of scene %d" % s) for s, ps in enumerate(items)])


def pack_bits(mask):
    """bool [B, nt] -> int32 [B, ceil(nt / 32)]: bit k % 32 of word k / 32 set iff mask[:, k]."""
    B, nt = mask.shape
    W = (nt + 31) // 32
    m = torch.zeros(B, 32 * W, dtype=torch.int64, device=mask.device)
    m[:, :nt] = mask.to(torch.int64)
    w = (m.reshape(B, W, 32) << torch.arange(32, device=mask.device)).sum(2)
    return torch.where(w >= 1 << 31, w - (1 << 32), w).to(torch.int32).contiguous()


def pixel_centres(height, width, lo, hi):
    """Centres of a height x width pixel grid over the window [lo, hi] (BatchedWorld.render): pixel (i, j) sits at
    (lo_x + (j + 1/2) (hi_x - lo_x) / width, lo_y + (i + 1/2) (hi_y - lo_y) / height), so row i grows with y (the
    reference's screen, gravity along +y). lo / hi [2] give [height * width, 2], [B, 2] give [B, height * width, 2],
    row-major (point i * width + j); differentiable in lo and hi."""
    j = torch.arange(width, dtype=lo.dtype, device=lo.device) + 0.5
    i = torch.arange(height, dtype=lo.dtype, device=lo.device) + 0.5
    span = hi - lo
    x = lo[..., 0:1] + j * span[..., 0:1] / width                                   # [..., W]
    y = lo[..., 1:2] + i * span[..., 1:2] / height                                  # [..., H]
    shape = lo.shape[:-1] + (height, width)
    grid = torch.stack([x.unsqueeze(-2).expand(shape), y.unsqueeze(-1).expand(shape)], -1)
    return grid.reshape(lo.shape[:-1] + (height * width, 2))


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
                 poly_mass=1.0, poly_fric=0.9, poly_rest=0.5, constraints=None, no_contact=None,
                 external_force=None, active=None, ccd=False):
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
        `obstacle_fric` / `obstacle_rest`: their friction / restitution, [B,no] or broadcastable.
        `constraints`: `Joint` / `FixedJoint` / `XConstraint` / `YConstraint` / `RotConstraint` specs naming dynamic
        bodies by index (topology shared by the batch); their equality rows follow the `static` pins' rows, in list
        order. `no_contact`: pairs (a, b) of indices in [circles, polygons, obstacles] that never make contact
        (Body.add_no_contact), shared by the batch, or a length-B list of such pair lists, one per scene; joints do not
        imply it. `external_force`: f(t) -> [B, nd, 3]
        (rot, x, y) given the per-scene time t [B], evaluated once per step at its start and added to gravity
        (ExternalForce); gradients reach whatever f closes over.
        `active`: bool [B, nb + npoly + no] (or broadcastable), which bodies of [circles, polygons, obstacles] take
        part in each scene, so that the scenes of one batch can hold different bodies (None: all of them). An inactive
        body is frozen: it gets no gravity and no external force, its p and v are carried through every step
        unchanged, and it makes no contact (the contact walk of each scene visits its active bodies only). A
        constraint belongs to the scenes in which all its bodies are active; one with active and inactive bodies in
        the same scene raises ValueError (list, e.g., a 4-link and a 7-link chain and activate one of them per scene).
        At most 8192 bodies in all (nb + npoly + no) with `active` or per-scene `no_contact`.
        `ccd`: continuous collision detection in `step()`: each scene's step ends at the first impact of its bodies'
        motion v dt (first_impact with gap eps / 2 and skip eps), so that a fast body does not pass through a thin one
        unseen; pairs already within eps are left to the contact solve. False (the default) steps as the reference."""
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
        self.cons = list(constraints) if constraints is not None else []
        self.external_force = external_force
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
        self.ccd = bool(ccd)
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
        # the walk over each scene's own bodies (lcpb200_contacts_active) when scenes differ in bodies or masks
        self.per_scene = active is not None or (no_contact is not None and per_scene_pairs(no_contact))
        if self.per_scene and nt > MAX_ACTIVE_BODIES:
            raise ValueError("BatchedWorld: with `active` or per-scene `no_contact` a world holds at most %d bodies "
                             "(nb + npoly + no), got %d" % (MAX_ACTIVE_BODIES, nt))
        ii, jj = torch.triu_indices(nt, nt, 1)
        if self.no:
            keep = ii < nd                                                          # obstacles never pair up
            ii, jj = ii[keep], jj[keep]
        self.pi, self.pj = ii.to(self.device), jj.to(self.device)                   # pair (i, j), i < j, lexicographic
        self.active, self.active_words = None, None          # active_words None: every body active in the walk
        if active is not None:
            self._init_active(active, nt)
            self.fext = torch.where(self.dof_active, self.fext, torch.zeros_like(self.fext))   # frozen: no gravity
        self._init_constraints(to)
        self.nc_mask, self.nc_stride = None, 0
        if no_contact is not None:
            self._init_no_contact(no_contact, nt)
        if self.np:
            # a polygon-polygon or polygon-obstacle pair may give 2 contacts
            most = int(self.pi.numel()) + int((self.pi >= nb).sum())
            self.cap = int(contact_capacity) if contact_capacity else max(1, min(most, (4 if self.no else 3) * nb + 8 * self.np))
        else:
            # a world of one circle has no pair but still needs one (unused) contact slot
            self.cap = int(contact_capacity) if contact_capacity else max(1, min(int(self.pi.numel()), (4 if self.no else 3) * nb))
        # 3 (nb + npoly) + 3 n_static <= 128 and <= 256 contacts: condensed-KKT kernels (fp32 / fp64,
        # differentiable); larger scenes: the banded large-scene kernels (fp64; lcp_banded.cuh)
        self.large = self.n + self.ne > 128 or 4 * self.cap > 1024
        if self.large and self.cons:
            # the banded kernel holds the equality rows and every body they touch in a border of <= 16 rows
            touched = set(self.static) | {k for c in self.cons for k in c.bodies()}
            border = 3 * len(touched) + self.ne
            if border > 16:
                raise ValueError("BatchedWorld: a large scene (3 (nb + npoly) + e > 128 or > 256 contacts) holds its "
                                 "equality rows and the bodies they touch in the banded kernel's border of at most 16 "
                                 "rows; here 3 x %d bodies + %d rows = %d" % (len(touched), self.ne, border))
        if self.large and (self.dtype != torch.float64 or self.ne > 16):
            raise ValueError("BatchedWorld: scenes with 3 (nb + npoly) + 3 n_static > 128 (or > 256 contacts) need "
                             "float64 and at most 5 pinned bodies (static obstacles do not count)")
        self.t = pos.new_zeros(B)
        self.find_contacts()
        if self.strict_no_pen and bool((self.max_penetration() > self.tol).any()):
            raise AssertionError("Interpenetration at start")                      # world.py:66-68

    # ------------------------------------------------------------------ constraints.py:13-173, world.py:156-170
    def _init_constraints(self, to):
        """Validates the constraint specs and sets up each Joint's state as Joint.__init__ does (constraints.py:16-27):
        pos = anchor, pos1 = anchor - pos(body1), (r1, rot1) = cart_to_polar(pos1). Adds their rows to self.ne."""
        nd, B = self.nd, self.B
        self._jstate = []                         # per constraint: [r1, rot1, pos1, pos] (Joint) or None
        for c in self.cons:
            if not isinstance(c, (Joint, FixedJoint, _AxisConstraint)):
                raise ValueError("constraints: expected Joint, FixedJoint, XConstraint, YConstraint or RotConstraint, "
                                 "got %r" % (c,))
            if isinstance(c, FixedJoint) and c.j is None:
                raise ValueError("constraints: FixedJoint needs two bodies")
            for k in (c.i,) + (() if c.j is None else (c.j,)):
                if not isinstance(k, int) or k < 0 or k >= nd + self.no:
                    raise ValueError("constraints: body index %r out of range (%d dynamic bodies)" % (k, nd))
                if k >= nd:
                    raise ValueError("constraints: body %d is an obstacle, which has no degrees of freedom (use "
                                     "j=None for a joint to a world point)" % k)
            if c.j is not None and c.i == c.j:
                raise ValueError("constraints: a constraint joins body %d to itself" % c.i)
            st = None
            if isinstance(c, Joint):
                a = to(c.anchor)
                if a.dim() == 1:
                    a = a.unsqueeze(0).expand(B, 2)
                if a.shape != (B, 2):
                    raise ValueError("constraints: Joint anchor must be [2] or [B, 2], got %s" % (tuple(a.shape),))
                if not bool(torch.isfinite(a.detach()).all()):
                    raise ValueError("constraints: non-finite Joint anchor")
                pos1 = a - self.p[:, c.i, 1:]
                r1, rot1 = _cart_to_polar(pos1)
                st = [r1, rot1, pos1, a]
            self._jstate.append(st)
            self.ne += c.num_constraints
        if self.cons:
            self.A = self._equality_rows()
        if self.active is not None:
            check_constraint_activity(self.cons, self.active)

    def _init_active(self, active, nt):
        """Per-scene body activity: self.active [B, nt] bool, body_active [B, nd, 1] / dof_active [B, n] for the
        freezing, and the bitmask of lcpb200_contacts_active, active_words [B, ceil(nt / 32)] (bit k of word k / 32)."""
        self.active = check_active(active, self.B, nt).to(self.device)
        self.body_active = self.active[:, :self.nd].unsqueeze(2)
        self.dof_active = self.body_active.expand(-1, -1, 3).reshape(self.B, self.n)
        self.active_words = pack_bits(self.active)

    def _equality_rows(self):
        """World.Je() (world.py:156-170) for every scene, [B, ne, n]: the `static` pins' identity rows, then each
        constraint's J() (constraints.py:29-36, :70-77, :106-108, :133-135, :160-162) at the current state, as
        differentiable torch ops."""
        B, n = self.B, self.n
        A = self.p.new_zeros(B, self.ne, n)
        for r, k in enumerate(self.static):
            for q in range(3):
                A[:, 3 * r + q, 3 * k + q] = 1.0
        r = 3 * len(self.static)
        for c, st in zip(self.cons, self._jstate):
            i, j = 3 * c.i, None if c.j is None else 3 * c.j
            if isinstance(c, _AxisConstraint):
                A[:, r, i + c.dof] = 1.0
            elif isinstance(c, Joint):
                pos1, pos = st[2], st[3]
                A[:, r, i], A[:, r, i + 1] = -pos1[:, 1], 1.0
                A[:, r + 1, i], A[:, r + 1, i + 2] = pos1[:, 0], 1.0
                if j is not None:
                    pos2 = pos - self.p[:, c.j, 1:]                       # update_pos: pos2 = pos - body2.pos
                    A[:, r, j], A[:, r, j + 1] = pos2[:, 1], -1.0
                    A[:, r + 1, j], A[:, r + 1, j + 2] = -pos2[:, 0], -1.0
            else:                                                          # FixedJoint: pos1 = 0, pos = body1.pos
                pos2 = self.p[:, c.i, 1:] - self.p[:, c.j, 1:]
                A[:, r, i + 1], A[:, r + 1, i + 2], A[:, r + 2, i] = 1.0, 1.0, 1.0
                A[:, r, j], A[:, r, j + 1] = pos2[:, 1], -1.0
                A[:, r + 1, j], A[:, r + 1, j + 2] = -pos2[:, 0], -1.0
                A[:, r + 2, j] = -1.0
            r += c.num_constraints
        return A

    def _move_joints(self, rot_start, vel, dts):
        """Joint.move(dt) after the bodies moved (constraints.py:38-49): rot1 = rot_start + v_rot(body1) dt,
        pos1 = polar_to_cart(r1, rot1), pos = pos(body1) + pos1. FixedJoint and the axis constraints keep no state."""
        for c, st, r0 in zip(self.cons, self._jstate, rot_start):
            if st is None:
                continue
            rot1 = r0 + vel[:, 3 * c.i] * dts
            pos1 = _polar_to_cart(st[0], rot1)
            pos = self.p[:, c.i, 1:] + pos1
            if self.active is not None:
                # a joint of frozen bodies keeps its state, as its bodies keep theirs
                on = self.active[:, c.i]
                rot1, pos1 = torch.where(on, rot1, st[1]), torch.where(on.unsqueeze(1), pos1, st[2])
                pos = torch.where(on.unsqueeze(1), pos, st[3])
            st[1:] = [rot1, pos1, pos]

    def _init_no_contact(self, pairs, nt):
        """Pair-exclusion bitmask (no_contact of lcpb200_contacts): bit i * nt + j (i < j) per excluded pair. A
        length-B list of pair lists gives one mask per scene ([B, words], nc_stride = words)."""
        words = no_contact_masks(pairs, self.B, nt)
        self.nc_mask = words.to(self.device)
        self.nc_stride = int(words.shape[1]) if words.dim() == 2 else 0
        self.nc_pair_excluded = mask_bits(self.nc_mask, nt, self.pi, self.pj)      # per pair of self.pi / self.pj

    # ------------------------------------------------------------------ contacts.py:60-292, batched
    def find_contacts(self):
        """Pair walk + ordered compaction on the GPU (lcpb200_contacts: the pairs of the body list [circles...,
        polygons..., obstacles...] of every scene in lexicographic order = the reference's contact order;
        circle-circle, circle-polygon and hull-hull rules, 0-2 contacts per pair; the `no_contact` pairs skipped),
        then the contact geometry of the selected pairs: from the same call when nothing needs autograd, else from
        torch ops (_geometry_torch, which rebuilds hull-hull contacts from the kernel's features), differentiable
        w.r.t. positions, radii, materials and the polygon / obstacle vertices."""
        lib = _lib.load()
        B, cap, dev, nb = self.B, self.cap, self.device, self.nb
        pverts = self.polygon_vertices() if self.np else None
        poly = (self.plocal, self.pfric, self.prest) if self.np else (None,) * 3
        obst = (self.ov, self.oref, self.ofric, self.orest) if self.no else (None,) * 4
        needs_graph = _needs_graph((self.p, self.rad, self.fric_coeff, self.restitution) + poly + obst)
        # feat selects the polygon walk, which worlds with polygons, no_contact pairs or per-scene bodies need; the
        # others keep the circle walk
        with_feat = self.np > 0 or self.nc_mask is not None or self.per_scene
        masks = (self.nc_mask, self.active_words) if self.per_scene else (self.nc_mask,)

        def walk(*ins):
            i32 = lambda *s_: torch.empty(*s_, dtype=torch.int32, device=dev)
            b1, b2, counts = i32(B, cap), i32(B, cap), i32(B)
            feat = i32(B, cap) if with_feat else None
            new = lambda *s_: torch.empty(B, cap, *s_, dtype=self.dtype, device=dev)
            geo = [None] * 6 if needs_graph else [new(2), new(2), new(2), new(), new(), new()]
            bodies = [_lib.ptr(t) for t in ins[:-len(masks)]]
            outs = [_lib.ptr(t) for t in (b1, b2, counts, feat, *geo)]
            with torch.cuda.device(dev):
                if self.per_scene:
                    _lib.check(lib.lcpb200_contacts_active(
                        _lib.dtype_code(self.dtype), B, nb, self.np, self.no, self.nv, cap, self.eps, *bodies, *outs,
                        _lib.ptr(ins[-2]), self.nc_stride, _lib.ptr(ins[-1]), _lib.stream_ptr(dev)))
                else:
                    _lib.check(lib.lcpb200_contacts(
                        _lib.dtype_code(self.dtype), B, nb, self.np, self.no, self.nv, cap, self.eps, *bodies, *outs,
                        _lib.ptr(ins[-1]), _lib.stream_ptr(dev)))
            # tensors only: _DetectFn marks every output non-differentiable
            return tuple(t for t in (b1, b2, counts, feat, *geo) if t is not None)
        pcen = self.p[:, nb:, 1:] if self.np else None
        ins = [_detached(t) for t in (self.p[:, :nb, 1:], self.rad, self.fric_coeff, self.restitution, pverts, pcen)
               + poly[1:] + obst]
        out = _detect(walk, *ins, *masks)
        b1, b2, counts = out[:3]
        feat = out[3] if with_feat else None
        if int(counts.max()) > cap:
            raise RuntimeError("BatchedWorld: a scene has %d contacts, capacity %d" % (int(counts.max()), cap))
        self.c_b1, self.c_b2, self.counts = b1, b2, counts
        if with_feat:
            self.c_feat = feat
        if not needs_graph:
            self.c_normal, self.c_p1, self.c_p2, self.c_pen, self.c_mu, self.c_rest = out[3 + with_feat:]
            return
        self.c_normal, self.c_p1, self.c_p2, pen, self.c_mu, self.c_rest = self._geometry_torch(b1, b2, feat, pverts)
        valid = torch.arange(cap, device=dev).unsqueeze(0) < counts.unsqueeze(1)
        self.c_pen = torch.where(valid, pen, pen.new_full((), -1e30))

    def polygon_vertices(self):
        """World-frame vertices [B, npoly, V, 2] of the dynamic polygons at the current p: centroid + R(rot) local
        (Hull.set_p / rotate_verts, bodies.py:202-214), differentiable in p and the polygons' initial vertices."""
        return self._vertices_at(self.p, self.plocal)

    def _vertices_at(self, p, plocal):
        """polygon_vertices() at the poses p [B', nd, 3] of polygons plocal [B', npoly, V, 2]"""
        q = p[:, self.nb:]
        c, s = torch.cos(q[:, :, 0:1]), torch.sin(q[:, :, 0:1])
        lx, ly = plocal[..., 0], plocal[..., 1]
        return torch.stack([q[:, :, 1:2] + (c * lx - s * ly), q[:, :, 2:3] + (s * lx + c * ly)], 3)

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
        cr, ci = _take2(ref, kr), _take2(ref, ki)
        vtx = lambda Vx, e: torch.gather(Vx, 2, e.unsqueeze(2).unsqueeze(3).expand(-1, -1, 1, 2)).squeeze(2)
        E = vtx(Vr, (re + 1) % V) - vtx(Vr, re)
        ln = E.norm(dim=2)
        n = _edge_normal(E, _orientation(Vr), torch.where(ln > 0, ln, torch.ones_like(ln)))   # of the reference edge
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
        E = torch.roll(V, -1, dims=2) - V
        ln = E.norm(dim=3)
        dg = ~(ln > 0)                                     # zero-length edges (repeated vertices): skipped, as the kernel
        # a length of 1 keeps the skipped entries finite, gradients too
        nrm = _edge_normal(E, _orientation(V).unsqueeze(2), torch.where(dg, torch.ones_like(ln), ln))
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
        circle-polygon: contacts.py:84-144, as lcpb200_contacts; hull-hull: _hull_torch, from the kernel's
        features feat), gradients reaching positions, radii, materials and the polygon / obstacle vertices.
        pverts: the dynamic polygons' world-frame vertices (worlds with polygons)."""
        nb = self.nb
        pos = self.p[:, :, 1:]
        i1, i2 = b1.long(), b2.long()
        take = lambda t, idx: torch.gather(t, 1, idx)
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
        elif self.no:
            polys, pref, pfr, prs = self.ov, self.oref, self.ofric, self.orest
        else:                                        # circles only (worlds with no_contact pairs)
            polys = None
        cc = i2 < nb
        j = torch.where(cc, i2, 0)
        k = torch.where(cc, 0, i2 - nb)
        c = _take2(pos, i1)
        r1 = take(self.rad, i1)
        one = torch.zeros_like(c)
        one[..., 0] = 1.0
        # circle-circle (slots of obstacle pairs and the padding pair (0, 0) of a one-body world get a harmless unit
        # offset: no 0 / 0 in either pass)
        dcc = torch.where((cc & (i1 != j)).unsqueeze(2), c - _take2(pos, j), one)
        dist = dcc.norm(dim=2)
        r2 = take(self.rad, j)
        pen_cc = r1 + r2 - dist
        n_cc = dcc / dist.unsqueeze(2)
        p1_cc = -n_cc * (r1 - pen_cc / 2).unsqueeze(2)
        p2_cc = n_cc * (r2 - pen_cc / 2).unsqueeze(2)
        if polys is None:
            return (n_cc, p1_cc, p2_cc, pen_cc, 0.5 * (take(self.fric_coeff, i1) + take(self.fric_coeff, j)),
                    0.5 * (take(self.restitution, i1) + take(self.restitution, j)))
        # circle-obstacle / circle-polygon
        inside, q, _, n_in, sep = self._circle_polygon_torch(c, k, polys)
        out = ~cc & ~inside
        dq = torch.where(out.unsqueeze(2), c - q, one)
        dq_n = dq.norm(dim=2)
        n_co = torch.where(inside.unsqueeze(2), n_in, dq / dq_n.unsqueeze(2))
        pen_co = torch.where(inside, r1 - sep, r1 - dq_n)
        q_co = torch.where(inside.unsqueeze(2), c - n_in * sep.unsqueeze(2), q)   # best_pt2 = center - n (dist + rad)
        p1_co = q_co - c
        p2_co = q_co - _take2(pref, k)
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
        independent implementation tests/test_gpu_world.py and tests/test_gpu_obstacles.py check lcpb200_contacts'
        circle walk against; pairs excluded per scene and pairs with an inactive body make no contact. Returns
        (counts, b1, b2). Not available for worlds with
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
            if self.nc_mask is not None:
                active = active & ~self.nc_pair_excluded                                  # contacts.py:60
            if self.active is not None:
                active = active & self.active[:, self.pi] & self.active[:, self.pj]
            counts = active.sum(1)
            order = torch.sort((~active).to(torch.int8), dim=1, stable=True)[1][:, :self.cap]
            return counts.to(torch.int32), self.pi[order].to(torch.int32), self.pj[order].to(torch.int32)
        d = pos[:, self.pi] - pos[:, self.pj]
        pen = self.rad[:, self.pi] + self.rad[:, self.pj] - d.norm(dim=2)
        active = pen >= -self.eps                                                  # `if penetration < -eps: return`
        if self.nc_mask is not None:
            active = active & ~self.nc_pair_excluded                                      # contacts.py:60
        if self.active is not None:
            active = active & self.active[:, self.pi] & self.active[:, self.pj]
        counts = active.sum(1)
        order = torch.sort((~active).to(torch.int8), dim=1, stable=True)[1][:, :self.cap]   # active pairs first, in pair order
        return counts.to(torch.int32), self.pi[order].to(torch.int32), self.pj[order].to(torch.int32)

    def max_penetration(self):
        return self.c_pen.max(dim=1)[0]

    # ------------------------------------------------------------------ ray casts
    def _float_arg(self, x, name):
        """x as a tensor of the world's dtype and device; a tensor must be floating-point."""
        if isinstance(x, torch.Tensor):
            if not x.is_floating_point():
                raise ValueError("%s: need a floating-point tensor, got dtype %s" % (name, x.dtype))
            return x.to(device=self.device, dtype=self.dtype)
        return torch.as_tensor(x, dtype=self.dtype, device=self.device)

    def _ray_arg(self, x, name):
        """A ray argument [B, R, 2] or [R, 2] (shared by the batch) as a [B, R, 2] tensor of the world's dtype / device."""
        x = self._float_arg(x, name)
        if x.dim() == 2:
            x = x.unsqueeze(0).expand(self.B, -1, -1)
        if x.dim() != 3 or x.shape[0] != self.B or x.shape[2] != 2 or x.shape[1] == 0:
            raise ValueError("%s: need [B, R, 2] or [R, 2] with R >= 1 (B = %d), got %s"
                             % (name, self.B, tuple(x.shape)))
        return x

    def _geometry_leaves(self):
        """The tensors the world's geometry is differentiated in (None where the world has none): p, the radii, the
        polygons' initial vertices and the obstacle vertices."""
        return self.p, self.rad, self.plocal if self.np else None, self.ov if self.no else None

    def _query(self, entry, queries, flags, n, max_dist, with_normal, pverts, no_contact=None, with_dist=False):
        """One call of the ray, point, body-distance or shape-cast kernel `entry` (lcpb200_raycast,
        lcpb200_signed_distance, lcpb200_body_distance or lcpb200_shapecast) over n queries per scene at the current
        state. The entry's arguments between overts and active_words are the tensors `queries` (None: NULL), then the
        ints `flags`. no_contact: for lcpb200_body_distance and lcpb200_shapecast, their arguments after active_words
        (the mask or None, its stride); those entries also write point_a (shapecast's point). pverts:
        polygon_vertices() (worlds with polygons). Returns (value [B, n], body [B, n] int64, feat [B, n] int32, normal
        [B, n, 2] when with_normal, else None, point_a [B, n, 2] with no_contact, else None). with_dist: the entry
        writes a second value [B, n] after feat (lcpb200_time_of_impact's dist), appended to the result."""
        lib = _lib.load()
        B, nb, dev = self.B, self.nb, self.device
        with_point = no_contact is not None

        def call(pos, rad, pv, ov, aw, nc, *qs):
            new = lambda *s_: torch.empty(B, n, *s_, dtype=self.dtype, device=dev)
            value = new()
            body = torch.empty(B, n, dtype=torch.int32, device=dev)
            feat = torch.empty(B, n, dtype=torch.int32, device=dev)
            normal = new(2) if with_normal else None
            point_a = new(2) if with_point else None
            value2 = new() if with_dist else None
            with torch.cuda.device(dev):
                _lib.check(getattr(lib, entry)(
                    _lib.dtype_code(self.dtype), B, nb, self.np, self.no, self.nv, n, max_dist, _lib.ptr(pos),
                    _lib.ptr(rad), _lib.ptr(pv), _lib.ptr(ov), *[_lib.ptr(q) for q in qs], *flags, _lib.ptr(aw),
                    *((_lib.ptr(nc), no_contact[1]) if with_point else ()), _lib.ptr(value), _lib.ptr(body),
                    _lib.ptr(feat), *((_lib.ptr(value2),) if with_dist else ()), _lib.ptr(normal),
                    *((_lib.ptr(point_a),) if with_point else ()), _lib.stream_ptr(dev)))
            # tensors only: _DetectFn marks every output non-differentiable
            return tuple(t for t in (value, body, feat, normal, point_a, value2) if t is not None)
        nc = no_contact[0] if with_point else None
        out = _detect(call, _detached(self.p[:, :nb, 1:]), _detached(self.rad), _detached(pverts),
                      _detached(self.ov if self.no else None), self.active_words, nc, *[_detached(q) for q in queries])
        rest = iter(out[3:])
        normal, point_a = next(rest) if with_normal else None, next(rest) if with_point else None
        if with_dist:
            return out[0], out[1].long(), out[2], normal, point_a, next(rest)
        return out[0], out[1].long(), out[2], normal, point_a

    def raycast(self, origin, direction, max_dist):
        """Casts rays against every scene's bodies at the current state (lcpb200_raycast): origin / direction
        [B, R, 2] or [R, 2] (shared by the batch); direction is normalised here. A ray hits a body only where it enters
        it within max_dist: an origin inside a body does not see that body. Returns (dist [B, R], body [B, R] int64
        indexing [circles, polygons, obstacles], -1 for no hit, normal [B, R, 2] at the hit); a ray that hits nothing
        reads max_dist with zero gradient and a zero normal, as does a zero or non-finite direction. Inactive bodies
        (`active`) are invisible.
        The kernel makes every discrete choice (which body, which edge). When a gradient or tangent is needed, dist and
        normal are rebuilt from those choices with torch ops, so that gradients reach the origins, the directions, p,
        the radii, the polygons' initial vertices and the obstacles' vertices (and forward_ad / torch.func work)."""
        o = self._ray_arg(origin, "origin")
        d = self._ray_arg(direction, "direction")
        if o.shape[1] != d.shape[1]:
            raise ValueError("direction: need as many rays as origin (%d), got %d" % (o.shape[1], d.shape[1]))
        md = _max_dist(max_dist)
        nrm = d.norm(dim=2, keepdim=True)
        u = d / torch.where(nrm > 0, nrm, torch.ones_like(nrm))      # a zero direction stays zero: it hits nothing
        pverts = self.polygon_vertices() if self.np else None
        needs_graph = _needs_graph((o, u) + self._geometry_leaves())
        dist, body, feat, normal, _ = self._query("lcpb200_raycast", (o, u), (), int(o.shape[1]), md, not needs_graph,
                                                    pverts)
        if needs_graph:
            dist, normal = self._ray_torch(o, u, body, feat.long(), md, pverts)
        return dist, body, normal

    def _ray_torch(self, x, u, body, feat, max_dist, pverts, rho=0.0):
        """Torch mirror of the cast primitive of csrc/lcp_raycast.cuh and csrc/lcp_shapecast.cuh, REBUILT FROM THE
        KERNEL'S CHOICES body / feat [B, K]: the ray x + t u (x, u [B, K, 2]) against the target inflated by rho ([B, K],
        or 0.0 for a ray cast). A circle (c, R) and a polygon vertex v (feat 256 + v, a circle (v, 0)): the entry
        t = k / (-b + sqrt(b^2 - k)) into the circle of radius R + rho and normal (w + t u) / (R + rho); a polygon face
        e (feat e < 256; raycast's entering edge): t = (n_e . (v_e - x) + rho) / n_e . u and normal n_e; max_dist (a
        constant) and a zero normal where nothing is hit. With rho = 0.0 the values are raycast's: R + 0.0 and
        s + 0.0 are exact."""
        nb = self.nb
        B, K = body.shape
        is_c = (body >= 0) & (body < nb)
        is_p = body >= nb
        is_v = is_p & (feat >= 256)
        is_f = is_p & ~is_v
        dist = torch.full((B, K), max_dist, dtype=x.dtype, device=x.device)
        normal = torch.zeros_like(x)
        polys = _polygons(pverts, self.ov if self.no else None) if self.np or self.no else None
        is_d = is_c | is_v                                     # a disk: a circle, or a vertex inflated by rho
        if nb or polys is not None:
            c = torch.zeros_like(x)
            R = torch.zeros_like(dist)
            if nb:
                ci = torch.where(is_c, body, 0)
                c = _take2(self.p[:, :nb, 1:], ci)
                R = torch.gather(self.rad, 1, ci)
            if polys is not None:
                vi = torch.where(is_v, (body - nb) * self.nv + feat - 256, 0)
                c = torch.where(is_v.unsqueeze(2), _take2(polys.reshape(B, -1, 2), vi), c)
                R = torch.where(is_v, torch.zeros_like(R), R)
            rr = R + rho
            w = x - c
            b = (u * w).sum(2)
            k = (w * w).sum(2) - rr * rr
            disc = torch.where(is_d, b * b - k, torch.ones_like(b))
            den = torch.where(is_d, -b + disc.sqrt(), torch.ones_like(b))
            t_c = k / den
            n_c = (w + t_c.unsqueeze(2) * u) / torch.where(is_d, rr, torch.ones_like(rr)).unsqueeze(2)
            dist = torch.where(is_d, t_c, dist)
            normal = torch.where(is_d.unsqueeze(2), n_c, normal)
        if polys is not None:
            ve, _, E, sg = _chosen_edge(polys, body, torch.where(is_v, 0, feat), nb)
            ln = E.norm(dim=2)
            n = _edge_normal(E, sg, torch.where(is_f, ln, torch.ones_like(ln)))
            den = (n * u).sum(2)
            t_p = ((n * (ve - x)).sum(2) + rho) / torch.where(is_f, den, -torch.ones_like(den))
            dist = torch.where(is_f, t_p, dist)
            normal = torch.where(is_f.unsqueeze(2), n, normal)
        return dist, normal

    def lidar(self, body, n_rays, max_dist, fov=2 * math.pi, start=0.0):
        """n_rays rays from the centre of dynamic body `body` (the same body in every scene), ray k at the angle
        p[:, body, 0] + start + k fov / n_rays: a lidar turning with its body. The mounting body, whose centre lies
        inside it, never appears in the readings. Returns what `raycast` returns."""
        if isinstance(body, bool) or not isinstance(body, int) or not 0 <= body < self.nd:
            raise ValueError("body: need the index of a dynamic body in [0, %d), got %r" % (self.nd, body))
        _check_count(n_rays, "n_rays")
        k = torch.arange(n_rays, dtype=self.dtype, device=self.device)
        ang = self.p[:, body, 0:1] + start + k * float(fov) / n_rays                           # [B, n_rays]
        direction = torch.stack([torch.cos(ang), torch.sin(ang)], 2)
        origin = self.p[:, body, 1:].unsqueeze(1).expand(-1, n_rays, -1)
        return self.raycast(origin, direction, max_dist)

    # ------------------------------------------------------------------ signed distances and images
    def signed_distance(self, points, max_dist):
        """Signed distance from query points to every scene's bodies at the current state (lcpb200_signed_distance):
        points [B, Q, 2], or [Q, 2] shared by the batch (read by every scene, not copied). Negative inside a body; the
        min over the scene's bodies (exact outside every body, a bound inside where bodies overlap). Returns (sdf [B, Q],
        body [B, Q] int64 indexing [circles, polygons, obstacles], -1 when no body lies within max_dist, normal [B, Q, 2],
        the unit direction in which the distance grows); a point with no body within max_dist, or a non-finite point,
        reads max_dist with zero gradient and a zero normal. Inactive bodies (`active`) are invisible.
        The kernel makes every discrete choice (which body, which edge, inside or outside). When a gradient or tangent
        is needed, sdf and normal are rebuilt from those choices with torch ops, so that gradients reach the points, p,
        the radii, the polygons' initial vertices and the obstacles' vertices (and forward_ad / torch.func work)."""
        return self._signed_distance(points, max_dist, True)

    def _signed_distance(self, points, max_dist, with_normal):
        x = self._float_arg(points, "points")
        shared = x.dim() == 2
        if not ((shared and x.shape[1] == 2 and x.shape[0] >= 1) or
                (x.dim() == 3 and x.shape[0] == self.B and x.shape[2] == 2 and x.shape[1] >= 1)):
            raise ValueError("points: need [B, Q, 2] or [Q, 2] with Q >= 1 (B = %d), got %s" % (self.B, tuple(x.shape)))
        md = _max_dist(max_dist)
        B, Q = self.B, int(x.shape[-2])
        if B * Q > 2 ** 31 - 1:
            raise ValueError("points: B * Q = %d exceeds int32 indexing" % (B * Q))
        pverts = self.polygon_vertices() if self.np else None
        needs_graph = _needs_graph((x,) + self._geometry_leaves())
        sdf, body, feat, normal, _ = self._query("lcpb200_signed_distance", (x,), (int(shared),), Q, md,
                                                 with_normal and not needs_graph, pverts)
        if needs_graph:
            sdf, normal = self._sdf_torch(x, body, feat.long(), md, pverts)
        return sdf, body, normal

    def _sdf_torch(self, points, body, feat, max_dist, pverts, cpos=None, rad=None, ov=None):
        """Torch mirror of csrc/lcp_sdf.cuh, REBUILT FROM THE KERNEL'S CHOICES body / feat [B, Q]: |x - c| - r and
        (x - c) / |x - c| for a circle; n_e . (x - v_e) and n_e inside a polygon (feat 256 + e); outside (feat e) the
        distance to the closest point q of edge e (v_e, v_f or v_e + t E) and (x - q) / |x - q|; max_dist (a constant)
        and a zero normal where no body was chosen. points [B, Q, 2] or [Q, 2]. A zero distance (a point at a circle's
        centre or on the closest point) gives a zero normal and finite gradients. cpos [B, nb, 2] / rad [B, nb] / ov
        [B, no, V, 2]: the circles' centres and radii and the obstacles' vertices, the world's when None."""
        nb = self.nb
        cpos = self.p[:, :nb, 1:] if cpos is None else cpos
        rad = self.rad if rad is None else rad
        ov = (self.ov if self.no else None) if ov is None else ov
        B, Q = body.shape
        x = points.expand(B, Q, 2) if points.dim() == 2 else points

        def length(d):
            """|d| and d / |d|, both 0 where d == 0 (no 0 / 0 in either pass)"""
            n2 = (d * d).sum(2)
            nz = n2 > 0
            ln = torch.where(nz, n2, torch.ones_like(n2)).sqrt()
            return torch.where(nz, ln, torch.zeros_like(ln)), torch.where(nz.unsqueeze(2), d / ln.unsqueeze(2),
                                                                          torch.zeros_like(d))
        is_c = (body >= 0) & (body < nb)
        is_p = body >= nb
        sdf = torch.full((B, Q), max_dist, dtype=x.dtype, device=x.device)
        normal = torch.zeros_like(x)
        if nb:
            ci = torch.where(is_c, body, 0)
            ln, n_c = length(x - _take2(cpos, ci))
            sdf = torch.where(is_c, ln - torch.gather(rad, 1, ci), sdf)
            normal = torch.where(is_c.unsqueeze(2), n_c, normal)
        if self.np or self.no:
            polys = _polygons(pverts, ov)
            inside = is_p & (feat >= 256)
            ve, vf, E, sg = _chosen_edge(polys, body, feat % 256, nb)
            ee = torch.where(is_p, (E * E).sum(2), torch.ones_like(E[..., 0]))
            n = _edge_normal(E, sg, ee.sqrt())
            w = x - ve
            t = ((w * E).sum(2) / ee).unsqueeze(2)
            q = torch.where(t <= 0, ve, torch.where(t >= 1, vf, ve + t * E))
            d_out, n_out = length(x - q)
            sdf = torch.where(inside, (n * w).sum(2), torch.where(is_p, d_out, sdf))
            normal = torch.where(inside.unsqueeze(2), n, torch.where(is_p.unsqueeze(2), n_out, normal))
        return sdf, normal

    def render(self, height, width, lo, hi, sigma=0.0, max_dist=None):
        """An image of every scene on a height x width pixel grid over the window [lo, hi] (pixel_centres: row i grows
        with y; lo = (0, 0), hi = (W, H) gives the reference's screen pixels). lo / hi [2] (one window for the batch) or
        [B, 2] (one per scene, e.g. following a body: lo = w.p[:, k, 1:] - 50); both may require grad.
        Returns (image [B, H, W], body [B, H, W] int64, sdf [B, H, W]) from signed_distance at the pixel centres:
        sigma > 0 gives the soft silhouette sigmoid(-sdf / sigma), differentiable like sdf; sigma == 0 the hard one
        (sdf <= 0) in the world's dtype, without gradient. body is the nearest body within max_dist (-1: none), so
        that any per-body attribute can be painted with it. max_dist None: the largest window diagonal (read on the
        host; pass max_dist explicitly under torch.func transforms)."""
        _check_count(height, "height")
        _check_count(width, "width")
        if self.B * height * width > 2 ** 31 - 1:
            raise ValueError("render: B * height * width = %d exceeds int32 indexing" % (self.B * height * width))
        sg = float(sigma)
        if not math.isfinite(sg) or sg < 0:
            raise ValueError("sigma: need a finite value >= 0, got %r" % (sigma,))
        win = []
        for name, v in (("lo", lo), ("hi", hi)):
            v = self._float_arg(v, name)
            if v.shape not in ((2,), (self.B, 2)):
                raise ValueError("%s: need [2] or [B, 2] (B = %d), got %s" % (name, self.B, tuple(v.shape)))
            win.append(v)
        lo, hi = win
        if lo.dim() != hi.dim():
            lo, hi = lo.expand(self.B, 2), hi.expand(self.B, 2)
        if not bool((lo.detach() < hi.detach()).all()):
            raise ValueError("render: need lo < hi in both coordinates")
        if max_dist is None:
            max_dist = float((hi.detach() - lo.detach()).norm(dim=-1).max())
        sdf, body, _ = self._signed_distance(pixel_centres(height, width, lo, hi), max_dist, False)
        image = torch.sigmoid(-sdf / sg) if sg > 0 else (sdf.detach() <= 0).to(self.dtype)
        shape = (self.B, height, width)
        return image.reshape(shape), body.reshape(shape), sdf.reshape(shape)

    # ------------------------------------------------------------------ distances between bodies
    def _body_arg(self, x, name, pair):
        """Body indices [K] / [B, K] (pair: [K, 2] / [B, K, 2]) indexing [circles, polygons, obstacles], as an int32
        tensor on the world's device; returns (indices, shared by the batch)."""
        t = x if isinstance(x, torch.Tensor) else torch.as_tensor(x)
        want = "[K, 2] or [B, K, 2]" if pair else "[K] or [B, K]"
        d = t.dim() - (1 if pair else 0)
        if d not in (1, 2) or (pair and t.shape[-1] != 2) or (d == 2 and t.shape[0] != self.B):
            raise ValueError("%s: need %s (B = %d), got %s" % (name, want, self.B, tuple(t.shape)))
        K = int(t.shape[d - 1])
        if K == 0:
            raise ValueError("%s: need K >= 1 queries, got %s" % (name, tuple(t.shape)))
        if t.dtype == torch.bool or t.is_floating_point() or t.is_complex():
            raise ValueError("%s: need integer body indices, got dtype %s" % (name, t.dtype))
        if self.B * K > 2 ** 31 - 1:
            raise ValueError("%s: B * K = %d exceeds int32 indexing" % (name, self.B * K))
        nt = self.nd + self.no
        lo, hi = int(t.min()), int(t.max())
        if lo < 0 or hi >= nt:
            raise ValueError("%s: body index %d out of range (%d bodies)" % (name, lo if lo < 0 else hi, nt))
        if pair and bool((t[..., 0] == t[..., 1]).any()):
            raise ValueError("%s: a pair names one body twice" % name)
        return t.to(device=self.device, dtype=torch.int32), d == 1

    def distance(self, pairs, max_dist):
        """Distance between the bodies of each pair at the current state (lcpb200_body_distance, pair mode): pairs
        [K, 2] (shared by the batch) or [B, K, 2] of indices into [circles, polygons, obstacles]. The rule (DESIGN.md
        section 8): the signed distance of one feature point of one body (a circle's centre minus its radius, or a
        polygon's vertex) to the other body; the exact Euclidean distance for separated bodies, and for overlapping
        polygons minus the minimum translation distance. Returns (dist [B, K], body [B, K] int64: the pair's second body,
        -1 when it is not within max_dist or a body is inactive, normal [B, K, 2]: the unit normal from the first body
        towards the second, point_a / point_b [B, K, 2]: the witnesses on the two bodies, point_b = point_a + dist
        normal). When separated the witnesses lie on the two boundaries; when overlapping one is the support vertex and
        the other its projection onto the supporting line of the separating face, which need not lie on the face
        segment. A miss reads max_dist, zero normal and witnesses, and zero gradient.
        The kernel makes every discrete choice (source point, target edge or face). When a gradient or tangent is
        needed, the outputs are rebuilt from those choices with torch ops (_distance_torch), so that gradients reach p,
        the radii, the polygons' initial vertices and the obstacles' vertices (and forward_ad / torch.func work)."""
        t, shared = self._body_arg(pairs, "pairs", True)
        return self._body_distance(t[..., 0], t[..., 1], shared, max_dist)

    def nearest(self, bodies, max_dist):
        """The nearest other body of each query body at the current state (lcpb200_body_distance, nearest mode):
        bodies [K] (shared by the batch) or [B, K] of indices into [circles, polygons, obstacles]. Candidates are every
        other active body of the scene, obstacles included, except the world's `no_contact` pairs (so that a link of a
        jointed chain does not read its neighbour at the joint); the lower index wins a tie. Returns what `distance`
        returns for the pair (query, nearest), with body the nearest body (-1: none within max_dist, or an inactive
        query body)."""
        t, shared = self._body_arg(bodies, "bodies", False)
        return self._body_distance(t, None, shared, max_dist)

    def _body_distance(self, ba, bb, shared, max_dist):
        md = _max_dist(max_dist)
        B, K = self.B, int(ba.shape[-1])
        pverts = self.polygon_vertices() if self.np else None
        needs_graph = _needs_graph(self._geometry_leaves())
        no_contact = (self.nc_mask, self.nc_stride) if bb is None else (None, 0)     # nearest mode only
        dist, body, feat, normal, point_a = self._query("lcpb200_body_distance", (ba, bb), (int(shared),), K, md, True,
                                                        pverts, no_contact)
        if needs_graph:
            dist, normal, point_a, point_b = self._distance_torch(ba.long().expand(B, K), body, feat.long(), md, pverts)
            return dist, body, normal, point_a, point_b
        return dist, body, normal, point_a, point_a + dist.unsqueeze(2) * normal

    def _distance_torch(self, ba, bo, feat, max_dist, pverts, cpos=None, rad=None, ov=None):
        """Torch mirror of csrc/lcp_distance.cuh, REBUILT FROM THE KERNEL'S CHOICES: ba [B, K] the first body, bo [B, K]
        the kernel's other body (-1: a miss), feat its packed choices. The source point x and radius r (a circle's
        centre and radius, or polygon vertex feat >> 9 & 255 and 0) of the source body (the other body iff bit 17),
        then one _sdf_torch of x against the target with the target feat (bits 0-8): d = sdf - r, n = -m (the first body
        the source) or m (the other), point_a = x - r m or x - sdf m, point_b = point_a + d n. A miss reads max_dist (a
        constant) and zeros. Returns (dist, normal, point_a, point_b). cpos / rad / ov: as in _sdf_torch."""
        nb = self.nb
        B, K = bo.shape
        cpos = self.p[:, :nb, 1:] if cpos is None else cpos
        rad = self.rad if rad is None else rad
        ov = (self.ov if self.no else None) if ov is None else ov
        hit = bo >= 0
        src_b = hit & (((feat >> 17) & 1) == 1)
        src = torch.where(src_b, bo, ba)
        tgt = torch.where(hit, torch.where(src_b, ba, bo), -1)
        is_c = src < nb
        dt = self.dtype
        x = torch.zeros(B, K, 2, dtype=dt, device=self.device)
        r = torch.zeros(B, K, dtype=dt, device=self.device)
        if nb:
            ci = torch.where(is_c, src, 0)
            x = _take2(cpos, ci)
            r = torch.where(is_c, torch.gather(rad, 1, ci), r)
        if self.np or self.no:
            polys = _polygons(pverts, ov)
            vi = torch.where(is_c | ~hit, 0, (src - nb) * self.nv + ((feat >> 9) & 255))   # a miss's feat is -1
            x = torch.where(is_c.unsqueeze(2), x, _take2(polys.reshape(B, -1, 2), vi))
        sdf, m = self._sdf_torch(x, tgt, feat & 511, max_dist, pverts, cpos, rad, ov)
        dist = torch.where(hit, sdf - r, sdf)
        normal = torch.where(src_b.unsqueeze(2), m, -m)
        w = torch.where(src_b, sdf, r)
        point_a = torch.where(hit.unsqueeze(2), x - w.unsqueeze(2) * m, torch.zeros_like(x))
        return dist, normal, point_a, point_a + dist.unsqueeze(2) * normal

    # ------------------------------------------------------------------ shape casts and sweeps
    def shapecast(self, origin, direction, radius, max_dist):
        """Sweeps disks against every scene's bodies at the current state (lcpb200_shapecast, disk mode): a disk of
        radius `radius` from `origin` along `direction` ([B, K, 2] or [K, 2] shared by the batch; direction is
        normalised here). radius: a scalar, [K] or [B, K], finite and >= 0. The disk hits a body where it first touches
        it within max_dist; a body the disk already overlaps at the origin is not seen (with radius 0 this is
        `raycast`). Returns (dist [B, K], body [B, K] int64 indexing [circles, polygons, obstacles], -1 for no hit,
        normal [B, K, 2]: the hit body's outward normal at the contact, point [B, K, 2]: the contact point on its
        surface, origin + dist u - radius normal); a miss reads max_dist, zeros and zero gradient, as does a zero or
        non-finite direction. Inactive bodies (`active`) are invisible.
        The kernel makes every discrete choice (which body, which face or vertex). When a gradient or tangent is
        needed, the outputs are rebuilt from those choices with torch ops, so that gradients reach the origins, the
        directions, the radii of the disks, p, the bodies' radii, the polygons' initial vertices and the obstacles'
        vertices (and forward_ad / torch.func work)."""
        o = self._ray_arg(origin, "origin")
        d = self._ray_arg(direction, "direction")
        K = int(o.shape[1])
        if d.shape[1] != K:
            raise ValueError("direction: need as many queries as origin (%d), got %d" % (K, d.shape[1]))
        r = self._float_arg(radius, "radius")
        if r.dim() == 0 or (r.dim() == 1 and r.shape[0] == K):
            r = r.expand(self.B, K)
        elif tuple(r.shape) != (self.B, K):
            raise ValueError("radius: need a scalar, [K] or [B, K] (B = %d, K = %d), got %s"
                             % (self.B, K, tuple(r.shape)))
        rd = r.detach()
        # the kernel reads a bad radius as a miss; it is rejected here wherever the values can be read
        if not torch._C._functorch.is_functorch_wrapped_tensor(rd) and not bool((torch.isfinite(rd) & (rd >= 0)).all()):
            raise ValueError("radius: need finite radii >= 0")
        md = _max_dist(max_dist)
        nrm = d.norm(dim=2, keepdim=True)
        u = d / torch.where(nrm > 0, nrm, torch.ones_like(nrm))      # a zero direction stays zero: it hits nothing
        pverts = self.polygon_vertices() if self.np else None
        needs_graph = _needs_graph((o, u, r) + self._geometry_leaves())
        dist, body, feat, normal, point = self._query("lcpb200_shapecast", (o, r, None, u, None), (), K, md, True,
                                                      pverts, (None, 0))
        if needs_graph:
            hit = body >= 0
            dist, normal = self._ray_torch(o, u, body, feat.long() & 511, md, pverts, r)
            point = torch.where(hit.unsqueeze(2), o + dist.unsqueeze(2) * u - r.unsqueeze(2) * normal,
                                torch.zeros_like(o))
        return dist, body, normal, point

    def sweep(self, bodies, displacement):
        """Translates each query body by `displacement` (no rotation) against every other body of its scene, held
        still, at the current state (lcpb200_shapecast, body mode): the continuous-collision question of how far a body
        can move before it touches something, e.g. sweep(ks, w.v.reshape(B, nd, 3)[:, ks, 1:] * w.dt). bodies [K]
        (shared by the batch) or [B, K] of indices into [circles, polygons, obstacles]; displacement [B, K, 2] or
        [K, 2]. Candidates are those of `nearest`: every other active body, obstacles included, except the world's
        `no_contact` partners of the mover. A body the mover already overlaps is not seen, one it touches is seen only
        when the motion heads into it: sweep reports new contacts, `distance` existing overlap.
        Returns (frac [B, K] in [0, 1]: the fraction of the displacement travelled at the first contact, 1 when nothing
        is hit, body [B, K] int64: the hit body, -1 for none (also for a zero displacement or an inactive mover),
        normal [B, K, 2]: the unit normal from the mover towards the hit body, point [B, K, 2]: the contact point in
        world coordinates at the time of impact); a miss reads frac 1, zeros and zero gradient.
        The kernel makes every discrete choice; when a gradient or tangent is needed the outputs are rebuilt from them
        with torch ops (_sweep_torch), so that gradients reach the displacement, p, the radii, the polygons' initial
        vertices and the obstacles' vertices (and forward_ad / torch.func work)."""
        bq, _ = self._body_arg(bodies, "bodies", False)
        d = self._ray_arg(displacement, "displacement")
        B, K = self.B, int(bq.shape[-1])
        if d.shape[1] != K:
            raise ValueError("displacement: need as many queries as bodies (%d), got %d" % (K, d.shape[1]))
        bq = bq.expand(B, K)
        L = d.norm(dim=2)
        Ls = torch.where(L > 0, L, torch.ones_like(L))
        u = d / Ls.unsqueeze(2)                                      # a zero displacement stays zero: it hits nothing
        pverts = self.polygon_vertices() if self.np else None
        needs_graph = _needs_graph((d,) + self._geometry_leaves())
        dist, body, feat, normal, point = self._query("lcpb200_shapecast", (None, None, bq, u, L), (), K, 0.0, True,
                                                      pverts, (self.nc_mask, self.nc_stride))
        if needs_graph:
            return self._sweep_torch(bq.long(), body, feat.long(), u, Ls, pverts)
        return torch.where(body >= 0, dist / Ls, torch.ones_like(dist)), body, normal, point

    def _sweep_torch(self, bq, bo, feat, u, L, pverts):
        """Torch mirror of lcpb200_shapecast's body mode, REBUILT FROM THE KERNEL'S CHOICES: bq [B, K] the movers, bo
        [B, K] the hit bodies (-1: a miss), feat their packed choices, u the unit directions, L the displacements'
        lengths (1 where zero). The source (the hit body iff bit 17) gives the point x and rho (a circle's centre and
        radius, or polygon vertex feat >> 9 & 255 and 0), cast along s u (s = -1 iff bit 17) against the target with
        the target feat (bits 0-8), one _ray_torch: frac = t / L, normal -m (or m when the mover is the target), point
        x + s t u - rho m, plus t u when the mover is the target. A miss reads frac 1 and zeros. Returns
        (frac, body, normal, point)."""
        nb = self.nb
        B, K = bo.shape
        hit = bo >= 0
        src_b = hit & (((feat >> 17) & 1) == 1)
        src = torch.where(src_b, bo, bq)
        tgt = torch.where(hit, torch.where(src_b, bq, bo), -1)
        is_c = src < nb
        dt = self.dtype
        x = torch.zeros(B, K, 2, dtype=dt, device=self.device)
        rho = torch.zeros(B, K, dtype=dt, device=self.device)
        if nb:
            ci = torch.where(is_c, src, 0)
            x = _take2(self.p[:, :nb, 1:], ci)
            rho = torch.where(is_c, torch.gather(self.rad, 1, ci), rho)
        if self.np or self.no:
            polys = _polygons(pverts, self.ov if self.no else None)
            vi = torch.where(is_c | ~hit, 0, (src - nb) * self.nv + ((feat >> 9) & 255))   # a miss's feat is -1
            x = torch.where(is_c.unsqueeze(2), x, _take2(polys.reshape(B, -1, 2), vi))
        su = torch.where(src_b.unsqueeze(2), -u, u)
        t, m = self._ray_torch(x, su, tgt, torch.where(hit, feat & 511, -1), 0.0, pverts, rho)
        frac = torch.where(hit, t / L, torch.ones_like(t))
        normal = torch.where(src_b.unsqueeze(2), m, -m)
        tu = torch.where(src_b, torch.zeros_like(t), t).unsqueeze(2) * u
        point = torch.where(hit.unsqueeze(2), x + tu - rho.unsqueeze(2) * m, torch.zeros_like(x))
        return frac, bo, normal, point

    # ------------------------------------------------------------------ times of impact
    def time_of_impact(self, pairs, motion, gap=0.0, skip=None, tol=None):
        """Time of impact of each pair of bodies, both translating and rotating over one motion, from the current state
        (lcpb200_time_of_impact, pair mode): pairs [K, 2] (shared by the batch) or [B, K, 2] of indices into [circles,
        polygons, obstacles]; motion [B, nd, 3] or [B, n], each dynamic body's displacement (rot, x, y) over the motion,
        e.g. w.v.reshape(B, nd, 3) * w.dt. Over tau in [0, 1] body k sits at p_k + tau motion_k (the motion of a
        step); obstacles stay. The first tau at which the pair's distance (`distance`) falls to `gap` is found by
        conservative advancement (DESIGN.md section 8), never later than the true contact; within `tol` (world units;
        default TOI_TOL of the dtype, 1e-9 in float64 and 1e-4 in float32). A pair closer than `skip` (default: gap) at
        tau = 0 is not seen, one exactly at skip only when it closes: new contacts, not existing ones.
        Returns (frac [B, K]: tau, 1 when nothing is hit, body [B, K] int64: the pair's second body, -1 for no hit, an
        inactive body or two still bodies, dist [B, K]: the distance at tau, normal [B, K, 2]: the unit normal from the
        first body towards the second at tau, point_a / point_b [B, K, 2]: the witnesses at tau, point_b = point_a +
        dist normal); a miss reads frac 1 and zeros, with zero gradient.
        The kernel makes every discrete choice; when a gradient or tangent is needed, the outputs are rebuilt from them
        with torch ops (_impact_torch): frac through the implicit-function derivative of the level set d = d(tau) at
        the hit, so that gradients reach the motion, p, the radii, the polygons' initial vertices and the obstacles'
        vertices (and forward_ad / torch.func work). A hit at tau = 0, or one where d does not fall (a grazing touch),
        carries no gradient of frac."""
        t, shared = self._body_arg(pairs, "pairs", True)
        return self._impact(t[..., 0], t[..., 1], shared, motion, gap, skip, tol)

    def first_impact(self, bodies, motion, gap=0.0, skip=None, tol=None):
        """The first impact of each query body over the motion (lcpb200_time_of_impact, first mode): bodies [K] (shared
        by the batch) or [B, K]; candidates are those of `nearest` (every other active body, obstacles included,
        except the world's `no_contact` partners), each moving by its own motion row; the lower index wins a tie.
        Returns what `time_of_impact` returns for the pair (query, first body hit)."""
        t, shared = self._body_arg(bodies, "bodies", False)
        return self._impact(t, None, shared, motion, gap, skip, tol)

    def _motion_arg(self, motion):
        """motion [B, nd, 3] or [B, n] as a [B, nd, 3] tensor of the world's dtype / device; finite where readable"""
        m = self._float_arg(motion, "motion")
        if tuple(m.shape) == (self.B, self.n):
            m = m.reshape(self.B, self.nd, 3)
        if tuple(m.shape) != (self.B, self.nd, 3):
            raise ValueError("motion: need [B, nd, 3] or [B, 3 nd] (B = %d, nd = %d), got %s"
                             % (self.B, self.nd, tuple(m.shape)))
        md = m.detach()
        # the kernel reads a non-finite row as no motion; it is rejected here wherever the values can be read
        if not torch._C._functorch.is_functorch_wrapped_tensor(md) and not bool(torch.isfinite(md).all()):
            raise ValueError("motion: need finite values")
        return m

    def _impact(self, ba, bb, shared, motion, gap, skip, tol):
        m = self._motion_arg(motion)
        gap = _length(gap, "gap")
        skip = gap if skip is None else _length(skip, "skip")
        tol = TOI_TOL[self.dtype] if tol is None else _length(tol, "tol")
        B, K = self.B, int(ba.shape[-1])
        pverts = self.polygon_vertices() if self.np else None
        pcen = self.p[:, self.nb:, 1:] if self.np else None
        needs_graph = _needs_graph((m,) + self._geometry_leaves())
        no_contact = (self.nc_mask, self.nc_stride) if bb is None else (None, 0)     # first mode only
        frac, body, feat, normal, point_a, dist = self._query(
            "lcpb200_time_of_impact", (pcen, m, ba, bb), (int(shared), skip, tol), K, gap, True, pverts, no_contact,
            with_dist=True)
        if needs_graph:
            return self._impact_torch(ba.long().expand(B, K), body, feat.long(), frac, m)
        return frac, body, dist, normal, point_a, point_a + dist.unsqueeze(2) * normal

    def _impact_torch(self, ba, bo, feat, tau, motion):
        """Torch mirror of lcpb200_time_of_impact, REBUILT FROM THE KERNEL'S CHOICES: ba [B, K] the first body, bo
        [B, K] the hit body (-1: a miss), feat the pair's distance choices at the kernel's tau [B, K], motion
        [B, nd, 3]. D(t) is _distance_torch of the pair at the poses p + t motion (each query at its own t). frac =
        tau - (D(tau) - D(tau).detach()) / Ddot, with tau and Ddot = n . (u_B(point_b) - u_A(point_a)) detached
        (u_k(x) = dc_k + dth_k perp(x - c_k(tau)), the velocity of body k's material point x; dth = 0 for a circle):
        the value is tau, the derivative that of the level set through the hit. Hits at tau = 0 or with Ddot >= 0 keep
        tau constant. dist, normal and the witnesses are D's at p + frac motion. A miss reads frac 1 and zeros.
        Returns (frac, body, dist, normal, point_a, point_b)."""
        nb, nd, no = self.nb, self.nd, self.no
        B, K = bo.shape
        hit = bo >= 0
        tau = tau.detach()
        circle = torch.zeros(nd, 1, dtype=torch.bool, device=motion.device)
        circle[:nb] = True
        mo = torch.cat([torch.where(circle, 0.0, motion[..., :1]), motion[..., 1:]], 2)   # a circle does not turn

        def at(t):
            """_distance_torch of every query at the poses p + t motion, t [B, K]; [B, K] / [B, K, 2] results"""
            p = (self.p.unsqueeze(1) + t.reshape(B, K, 1, 1) * mo.unsqueeze(1)).reshape(B * K, nd, 3)
            rep = lambda x: None if x is None else x.repeat_interleave(K, 0)
            pv = self._vertices_at(p, rep(self.plocal)) if self.np else None
            ov = rep(self.ov) if no else None
            out = self._distance_torch(ba.reshape(-1, 1), bo.reshape(-1, 1), feat.reshape(-1, 1), 0.0, pv,
                                       p[:, :nb, 1:], rep(self.rad), ov)
            return [x.reshape((B, K) + x.shape[2:]) for x in out]
        d, n, pa, pb = at(tau)
        # the velocities of the witnesses, detached; obstacles (index >= nd) do not move
        full = torch.cat([mo, mo.new_zeros(B, no, 3)], 1).detach()
        cen = torch.cat([self.p[..., 1:], self.p.new_zeros(B, no, 2)], 1).detach()

        def vel(k, x):
            dk = torch.gather(full, 1, k.unsqueeze(2).expand(-1, -1, 3))
            w = x.detach() - (_take2(cen, k) + tau.unsqueeze(2) * dk[..., 1:])
            return dk[..., 1:] + dk[..., :1] * torch.stack([-w[..., 1], w[..., 0]], 2)
        ddot = (n.detach() * (vel(torch.where(hit, bo, 0), pb) - vel(ba, pa))).sum(2)
        moving = hit & (tau > 0) & (ddot < 0)
        frac = tau - torch.where(moving, (d - d.detach()) / torch.where(moving, ddot, torch.ones_like(ddot)),
                                 torch.zeros_like(d))
        dist, normal, point_a, point_b = at(frac)
        return frac, bo, dist, normal, point_a, point_b

    # ------------------------------------------------------------------ engine calls
    def _lcp(self, mode, dt, b, fext=None):
        mass, inertia, v = self.mass, self.inertia, self.v
        if self.active is not None:
            # frozen bodies are isolated blocks of K whose results step_dt discards: no gradient through them
            keep = lambda t, m: torch.where(m, t, t.detach())
            mass, inertia = keep(mass, self.body_active[..., 0]), keep(inertia, self.body_active[..., 0])
            v = keep(v, self.dof_active)
        z, status = engine_solve(mass, inertia, v, self.fext if fext is None else fext, self.c_normal,
                                 self.c_p1, self.c_p2, self.c_mu, self.c_rest, self.c_b1, self.c_b2, dt, A=self.A, b=b,
                                 mode=mode,
                                 max_iter=self.max_iter if mode == 0 else 10, exact_adjoint=self.exact_adjoint,
                                 counts=self.counts)
        if bool((status == _lib.STATUS_SINGULAR_Q).any()):
            from .lcp import SINGULAR_Q_MSG
            raise RuntimeError(SINGULAR_Q_MSG)
        if bool((status == -100).any()):
            raise RuntimeError("BatchedWorld: a scene's contact topology is not supported by the fused kernel")
        return z

    def solve_dynamics(self, dt):
        """engines.py:26-78 for every scene: new_v = -zhat. The constraints' rows are rebuilt at the current state and
        the external force is evaluated at the step's start time (apply_forces(world.t), engines.py:27-32)."""
        if self.cons:
            self.A = self._equality_rows()
        b = self.v.new_zeros(self.B, self.ne) if self.ne else None
        fext = None
        if self.external_force is not None:
            f = self.external_force(self.t)
            if tuple(f.shape) != (self.B, self.nd, 3):
                raise ValueError("external_force: f(t) must return [B, nd, 3] = %s, got %s"
                                 % ((self.B, self.nd, 3), tuple(f.shape)))
            f = f.reshape(self.B, self.n)
            if self.active is not None:
                f = torch.where(self.dof_active, f, torch.zeros_like(f))
            fext = self.fext + f
        return -self._lcp(0, dt, b, fext)

    def post_stabilization(self):
        """engines.py:80-116 for every scene: -zhat with b = Je v, the constraints' rows at the current pose."""
        if self.cons:
            self.A = self._equality_rows()
        b = torch.bmm(self.A, self.v.unsqueeze(2)).squeeze(2) if self.ne else None
        return -self._lcp(1, 0.0, b)

    # ------------------------------------------------------------------ world.py:72-122
    def step(self):
        self.step_dt(self.dt)

    def step_dt(self, dt):
        start_p = self.p.clone()
        start_rot = [st[1] if st is not None else None for st in self._jstate]      # world.py:85
        start_v = self.v
        self.v = self.solve_dynamics(dt)
        if self.active is not None:
            self.v = torch.where(self.dof_active, self.v, start_v)                 # frozen bodies keep p and v
        if self.ccd:
            # end the step at the first impact: the pair then sits near eps / 2, inside the contact margin eps
            dyn = torch.arange(self.nd, device=self.device)
            toi = self.first_impact(dyn, self.v.reshape(self.B, self.nd, 3) * float(dt), gap=self.eps / 2,
                                    skip=self.eps)[0]
            dts = float(dt) * toi.min(dim=1).values
        else:
            dts = self.v.new_full((self.B,), float(dt))
        done = torch.zeros(self.B, dtype=torch.bool, device=self.device)
        while True:
            moved = start_p + self.v.reshape(self.B, self.nd, 3) * dts.reshape(self.B, 1, 1)      # body.move(dt)
            if self.active is not None:
                moved = torch.where(self.body_active, moved, start_p)
            self.p = torch.where(done.reshape(self.B, 1, 1), self.p, moved)
            self.find_contacts()
            ok = self.max_penetration() <= self.tol
            if not self.strict_no_pen:
                ok = ok | (dts < self.dt / 4)                                      # world.py:98-100
            done = done | ok
            if bool(done.all()):
                break
            dts = torch.where(done, dts, dts / 2)                                  # world.py:101 (positions reset: start_p)
        if self.cons:
            # joints moved with the bodies by the step's final dt, from the start value (world.py:92-93, :104-107)
            self._move_joints(start_rot, self.v, dts)
        if self.post_stab:
            tmp_v = self.v
            dp = self.post_stabilization() / 2                                     # world.py:111-112
            if self.active is not None:
                dp = torch.where(self.dof_active, dp, torch.zeros_like(dp))
            self.p = self.p + dp.reshape(self.B, self.nd, 3) * dts.reshape(self.B, 1, 1)
            if self.cons:
                self._move_joints([st[1] if st is not None else None for st in self._jstate], dp, dts)   # :117-118
            self.v = tmp_v
            self.find_contacts()
        self.t = self.t + dts

    def get_v(self):
        return self.v

    def get_p(self):
        return self.p.reshape(self.B, self.n)

    # ------------------------------------------------------------------ Jacobian of a step
    def linearize(self, chunk_size=None):
        """The Jacobian of one `step()` from the current state, per scene: returns (x_next [B, 2n], A [B, 2n, 2n],
        Bu [B, 2n, n]) with x = (get_p(), v) and x_next = f(x, u) the state after the step. u is an additive
        generalised force on the n dofs for this step (zero here; it enters like `external_force`). Rows of A and Bu:
        p' then v'. What model-predictive control, iLQR and Gauss-Newton identification linearise around.

        It is the Jacobian of the branch `step()` takes: the contact set, each scene's dt-halving count and the hull
        features are those of the step from this state, held fixed. Post-stabilisation, constraints, `no_contact`,
        obstacles, polygons and `external_force` are included; the internal state of a `Joint` (its anchor angle) is
        held fixed and is not part of x. Gradients through the LCP follow `exact_adjoint`: with friction on, only
        exact_adjoint=True gives the true derivative (DESIGN.md section 3.4).

        One `torch.func.vjp` of the step, then a `vmap` over the 2n one-hot cotangents (each placed in every scene at
        once: scenes are independent), `chunk_size` of them per pass (all at once by default; smaller chunks bound the
        memory). Each pass factors every scene's KKT matrix once for all of its cotangents. The world is left as it
        was (state, joints, contact list); only `last_solve_info()` then describes the linearisation's solves."""
        B, n = self.B, self.n
        saved = dict(self.__dict__)
        saved_joints = [None if st is None else list(st) for st in self._jstate]
        ef = self.external_force
        x0 = torch.cat([self.get_p(), self.v], 1).detach()

        def f(x, u):
            self.p = x[:, :n].reshape(B, self.nd, 3)
            self.v = x[:, n:]
            ub = u.reshape(B, self.nd, 3)
            self.external_force = (lambda t: ub) if ef is None else (lambda t: ef(t) + ub)
            self.find_contacts()                              # the contact geometry as a function of p
            self.step_dt(self.dt)
            return torch.cat([self.get_p(), self.v], 1)

        try:
            x_next, vjp_fn = torch.func.vjp(f, x0, x0.new_zeros(B, n))
            eye = torch.eye(2 * n, dtype=x0.dtype, device=x0.device).unsqueeze(1).expand(-1, B, -1)
            ja, jb = torch.func.vmap(vjp_fn, chunk_size=chunk_size)(eye)          # [2n, B, 2n], [2n, B, n]
        finally:
            self.__dict__.clear()
            self.__dict__.update(saved)
            for st, old in zip(self._jstate, saved_joints):            # the step moved the joints in place
                if st is not None:
                    st[:] = old
        return x_next.detach(), ja.transpose(0, 1).contiguous(), jb.transpose(0, 1).contiguous()
