"""Float64 host restatement of the contact walk of csrc/lcp_contacts.cuh (lcpb200_contacts), no GPU.

* `pair_list` restates the walk's enumeration: pairs (i, j), i < j, i a dynamic body (circle or polygon), in
  lexicographic order; obstacles never pair with each other.
* `scene_contacts` restates one scene's walk and geometry: the `no_contact` mask (only bits with i < j are read),
  the circle-circle rule (vectorised), the circle-polygon rule (`oracle.obstacle_oracle.circle_polygon`) and the
  hull-hull rule (`oracle.polygon_oracle`: `separations`, `get_incident_edge`, `clip_segment_to_line`), with the
  hull-hull features `feat` derived from the same choices (reference and incident edge, which body holds the
  reference face, the first clip's outcome, the clipped point). It also reports the smallest decision margin of
  the scene: how close any rule's quantity came to its threshold or tie, which bounds where a float32 walk may
  decide differently.
* `truncate` applies the capacity: the first `cap` contacts, padding with the pair (0, 1) ((0, 0) for one body),
  feat -1 (0 when there are no circles) and penetration -1e30; the count stays the true count.
* Scene builders: all-contact scenes (every pair is a contact), random mixed scenes, axis-aligned stacks with exact
  ties, regular 256-gons and scenes that sit exactly on each rule's inclusive boundary.

A scene is a dict of float64 numpy arrays: pos [nb, 2], rad / fric / rest [nb], pverts [np, nv, 2] (positive
area), pcen [np, 2], pfric / prest [np], overts [no, nv, 2] (either orientation), oref [no, 2], ofric / orest [no].
A batch is the same dict with a leading batch dimension.
"""
import itertools
import math

import numpy as np
import torch

from oracle.obstacle_oracle import circle_polygon
from oracle.polygon_oracle import clip_segment_to_line, get_incident_edge, left_orthogonal, separations

CHUNK = 256 * 4                 # pairs one CTA walks per chunk (NT * ITEMS)
MAX_NV = 256
PAD_PEN = -1e30
KEYS = ("pos", "rad", "fric", "rest", "pverts", "pcen", "pfric", "prest", "overts", "oref", "ofric", "orest")


# ---------------------------------------------------------------------------------------------------- enumeration
def n_pairs(nb, npoly, no):
    nd = nb + npoly
    return nd * (2 * (nd + no) - nd - 1) // 2


def pair_list(nb, npoly, no):
    """(I, J) int64 arrays of the walk's pairs in its order."""
    nd, nt = nb + npoly, nb + npoly + no
    if nd == 0 or nt < 2:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    rows = [np.full(nt - 1 - i, i, np.int64) for i in range(nd)]
    cols = [np.arange(i + 1, nt, dtype=np.int64) for i in range(nd)]
    return np.concatenate(rows), np.concatenate(cols)


def pair_list_itertools(nb, npoly, no):
    nd, nt = nb + npoly, nb + npoly + no
    return [(i, j) for i, j in itertools.combinations(range(nt), 2) if i < nd]


def row_starts(nb, npoly, no):
    """index of the first pair of every row i < nd"""
    nd, nt = nb + npoly, nb + npoly + no
    return [i * (2 * nt - i - 1) // 2 for i in range(nd)]


def shape_for_pairs(P, no_max=64):
    """(nb, no) with nb (nb - 1) / 2 + nb no == P: the largest nb with 0 < no <= no_max, else one circle and P
    obstacles (a power of two has no other shape)"""
    for nb in range(int(math.isqrt(2 * P)) + 1, 1, -1):
        rest = P - nb * (nb - 1) // 2
        if rest > 0 and rest % nb == 0 and rest // nb <= no_max:
            return nb, rest // nb
    return 1, P


# ---------------------------------------------------------------------------------------------------- mask
def mask_words(nt, pairs):
    """uint32 words of the no_contact mask with bit a * nt + b set for every (a, b) in pairs (any order of a, b is
    written as given: bits with a >= b are set too, which the walk must ignore)"""
    w = np.zeros((nt * nt + 31) // 32, dtype=np.uint32)
    for a, b in pairs:
        bit = a * nt + b
        w[bit >> 5] |= np.uint32(1 << (bit & 31))
    return w


def mask_bits(words, I, J, nt):
    bit = I * nt + J
    return ((words[bit >> 5] >> (bit & 31).astype(np.uint32)) & 1).astype(bool)


# ---------------------------------------------------------------------------------------------------- rules
def pack_feat(kind, clip1, ref2, re, ie):
    return kind | clip1 << 2 | ref2 << 4 | re << 5 | ie << 13


def unpack_feat(f):
    return dict(kind=f & 3, clip1=(f >> 2) & 3, ref2=(f >> 4) & 1, re=(f >> 5) & 255, ie=(f >> 13) & 255)


def circle_circle(pos, rad, I, J):
    """contacts.py:69-77 for pairs of circles, vectorised: (pen, normal, p1, p2)"""
    d = pos[I] - pos[J]
    dist = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1])
    pen = rad[I] + rad[J] - dist
    with np.errstate(invalid="ignore", divide="ignore"):
        n = d / dist[:, None]
    p1 = -n * (rad[I] - pen / 2)[:, None]
    p2 = n * (rad[J] - pen / 2)[:, None]
    return pen, n, p1, p2


def _orient(P):
    area = float(np.sum(P[:, 0] * np.roll(P, -1, 0)[:, 1] - P[:, 1] * np.roll(P, -1, 0)[:, 0]))
    return 1.0 if area > 0 else -1.0


def _circle_poly(c, r, P, ref, eps, marg):
    """contacts.py:84-144 through oracle.obstacle_oracle.circle_polygon: None or (normal, p1, p2, pen)"""
    t = torch.from_numpy
    hit = circle_polygon(t(c), t(P))
    E = np.roll(P, -1, 0) - P
    ln = np.sqrt((E * E).sum(1))
    ok = ln > 0
    o = _orient(P)
    nrm = o * np.stack([E[ok, 1], -E[ok, 0]], 1) / ln[ok, None]
    sp = (nrm * (c - P[ok])).sum(1)
    marg.append(abs(float(sp.max())))                      # inside / outside
    if hit[0] == "out":
        q = hit[1].numpy()
        dist = float(np.linalg.norm(c - q))
        marg.append(abs(dist - r - eps))
        if dist - r > eps:
            return None
        n = (c - q) / dist
        pen = r - dist
    else:
        n, s = hit[1].numpy(), float(hit[2])
        srt = np.sort(sp)
        if len(srt) > 1:
            marg.append(float(srt[-1] - srt[-2]))          # the separating edge
        q = c - n * s
        pen = r - s
    return n, q - c, q - ref, pen


def _hull_hull(V1, c1, V2, c2, eps, marg):
    """contacts.py:145-201 through oracle.polygon_oracle for world-frame vertices V1 / V2 and centroids c1 / c2:
    [(feat, normal, p1, p2, pen)]"""
    t = torch.from_numpy
    nv = V1.shape[0]
    v1, v2 = [t(v - c1) for v in V1], [t(v - c2) for v in V2]
    p1, p2 = t(c1), t(c2)
    s1 = separations(v1, p1, v2, p2, eps)
    if s1[0] > eps:
        marg.append(s1[0] - eps)
        return []
    s2 = separations(v2, p2, v1, p1, eps)
    if s2[0] > eps:
        marg.append(s2[0] - eps)
        return []
    marg += [eps - s1[0], eps - s2[0], abs(s2[0] - s1[0])]
    ref2 = s2[0] > s1[0]
    dist_, normal, sup, edge_norm, re, m = s2 if ref2 else s1
    marg.append(m)                                             # SAT winner over runner-up
    vr, pr, vi, pin, Vi = (v2, p2, v1, p1, V1) if ref2 else (v1, p1, v2, p2, V2)
    # support vertex: winner over the runner-up among distinct points
    dots = -(Vi - (c1 if ref2 else c2)) @ normal.numpy()
    best = dots[sup]
    others = [dots[k] for k in range(nv) if not np.array_equal(Vi[k], Vi[sup])]
    if others:
        marg.append(float(best - max(others)))
    ie = get_incident_edge(normal, vi, sup)
    # incident edge: the two candidates' dot products
    o = _orient(Vi)
    ok = lambda e: np.linalg.norm(Vi[(e + 1) % nv] - Vi[e]) > 0
    prev = next(e for e in ((sup - k) % nv for k in range(1, nv + 1)) if ok(e))
    nxt = next(e for e in ((sup + k) % nv for k in range(nv)) if ok(e))
    dn = []
    for e in (prev, nxt):
        E = Vi[(e + 1) % nv] - Vi[e]
        dn.append(float(normal.numpy() @ (o * np.array([E[1], -E[0]]) / np.linalg.norm(E))))
    if prev != nxt:
        marg.append(abs(dn[0] - dn[1]))
    incident = [vi[ie] + pin - pr, vi[(ie + 1) % nv] + pin - pr]
    cp = left_orthogonal(normal)
    h = edge_norm / 2
    d0, d1 = float(cp.dot(incident[0]) + h), float(cp.dot(incident[1]) + h)
    marg += [abs(d0), abs(d1)]
    clip1 = (0 if d1 >= 0 else 1) if d0 >= 0 else (2 if d1 >= 0 else 3)
    clipped = clip_segment_to_line(incident, cp, h)
    if len(clipped) < 2:
        assert clip1 == 3
        return []
    la, lb = {0: (0, 1), 1: (0, 2), 2: (1, 2)}[clip1]
    e0, e1 = float(-cp.dot(clipped[0]) + h), float(-cp.dot(clipped[1]) + h)
    marg += [abs(e0), abs(e1)]
    kinds = ([la] if e0 >= 0 else []) + ([lb] if e1 >= 0 else [])
    if e0 * e1 < 0 or len(kinds) < 2:
        kinds.append(3)
    clipped = clip_segment_to_line(clipped, -cp, h)
    assert len(clipped) == len(kinds)
    out = []
    for v, kind in zip(clipped, kinds):
        dist = normal.dot(v - vr[re])
        marg.append(abs(float(dist) - eps))
        if float(dist) <= eps:
            pt1 = v + normal * -dist
            pt2 = pt1 + pr - pin
            g = (normal, pt2, pt1) if ref2 else (-normal, pt1, pt2)
            out.append((pack_feat(kind, clip1, int(ref2), re, ie),) + tuple(x.numpy() for x in g) + (-float(dist),))
    return out


# ---------------------------------------------------------------------------------------------------- one scene
def scene_of(batch, s):
    return {k: batch[k][s] for k in KEYS}


def scene_contacts(sc, eps, mask=None):
    """The walk of one scene: dict(b1, b2, feat, normal, p1, p2, pen, mu, rest) in contact order (float64 numpy),
    count, and margin (the smallest decision margin, inf without decisions)."""
    nb, npoly, no = sc["pos"].shape[0], sc["pverts"].shape[0], sc["overts"].shape[0]
    nt = nb + npoly + no
    I, J = pair_list(nb, npoly, no)
    if mask is not None:
        keep = ~mask_bits(mask, I, J, nt)
        I, J = I[keep], J[keep]
    verts = lambda b: sc["pverts"][b - nb] if b < nb + npoly else sc["overts"][b - nb - npoly]
    cen = lambda b: sc["pcen"][b - nb] if b < nb + npoly else sc["oref"][b - nb - npoly]
    fr = np.concatenate([sc["fric"], sc["pfric"], sc["ofric"]])
    rs = np.concatenate([sc["rest"], sc["prest"], sc["orest"]])
    marg = []
    cc = J < nb
    cnt = np.zeros(I.shape[0], np.int64)
    pen_cc, n_cc, p1_cc, p2_cc = circle_circle(sc["pos"], sc["rad"], I[cc], J[cc])
    hit_cc = ~(pen_cc < -eps)
    if cc.any():
        marg.append(float(np.abs(pen_cc + eps).min()))
    cnt[cc] = hit_cc
    other = {}
    for q in np.nonzero(~cc)[0]:
        i, j = int(I[q]), int(J[q])
        if i < nb:
            g = _circle_poly(sc["pos"][i], float(sc["rad"][i]), verts(j), cen(j), eps, marg)
            res = [] if g is None else [(-1,) + g]
        else:
            res = _hull_hull(verts(i), cen(i), verts(j), cen(j), eps, marg)
        other[q] = res
        cnt[q] = len(res)
    n = int(cnt.sum())
    off = np.cumsum(cnt) - cnt
    out = dict(b1=np.repeat(I, cnt), b2=np.repeat(J, cnt), feat=np.full(n, -1, np.int64), normal=np.zeros((n, 2)),
               p1=np.zeros((n, 2)), p2=np.zeros((n, 2)), pen=np.zeros(n))
    qc = np.nonzero(cc)[0][hit_cc]
    for k, a in (("normal", n_cc), ("p1", p1_cc), ("p2", p2_cc), ("pen", pen_cc)):
        out[k][off[qc]] = a[hit_cc]
    for q, res in other.items():
        for u, (f, nrm, a1, a2, pn) in enumerate(res):
            at = off[q] + u
            out["feat"][at], out["normal"][at], out["p1"][at], out["p2"][at], out["pen"][at] = f, nrm, a1, a2, pn
    out["mu"] = 0.5 * (fr[out["b1"]] + fr[out["b2"]])
    out["rest"] = 0.5 * (rs[out["b1"]] + rs[out["b2"]])
    out["count"] = n
    out["margin"] = min(marg) if marg else math.inf
    return out


def truncate(res, cap, nb, nt):
    """The walk's outputs for capacity cap: b1 / b2 / feat [cap] int64 and pen [cap] with the padding, and the true
    count."""
    n = min(res["count"], cap)
    b1, b2 = np.zeros(cap, np.int64), np.full(cap, 1 if nt > 1 else 0, np.int64)
    feat = np.full(cap, 0 if nb == 0 else -1, np.int64)
    pen = np.full(cap, PAD_PEN)
    b1[:n], b2[:n], feat[:n], pen[:n] = res["b1"][:n], res["b2"][:n], res["feat"][:n], res["pen"][:n]
    return dict(b1=b1, b2=b2, feat=feat, pen=pen, count=res["count"])


# ---------------------------------------------------------------------------------------------------- scenes
def centroid(V):
    """area centroid of polygons [..., nv, 2] (repeated vertices allowed), float64"""
    a, b = V, np.roll(V, -1, axis=-2)
    cr = b[..., 0] * a[..., 1] - b[..., 1] * a[..., 0]
    return (cr[..., None] * (a + b)).sum(-2) / (6 * (cr.sum(-1) / 2)[..., None])


def make_scene(pos=None, rad=None, pverts=None, overts=None, nv=4, seed=0):
    """a scene dict from circles (pos [nb, 2], rad [nb]), dynamic polygons [np, nv, 2] and obstacles [no, nv, 2];
    materials drawn from `seed`"""
    g = np.random.default_rng(seed)
    pos = np.zeros((0, 2)) if pos is None else np.asarray(pos, np.float64).reshape(-1, 2)
    nb = pos.shape[0]
    rad = np.zeros(0) if rad is None else np.broadcast_to(np.asarray(rad, np.float64), (nb,)).copy()
    pv = np.zeros((0, nv, 2)) if pverts is None else np.asarray(pverts, np.float64)
    ov = np.zeros((0, nv, 2)) if overts is None else np.asarray(overts, np.float64)
    u = lambda n: np.round(0.1 + 0.8 * g.random(n), 3)
    return dict(pos=pos, rad=rad, fric=u(nb), rest=u(nb), pverts=pv, pcen=centroid(pv) if len(pv) else np.zeros((0, 2)),
                pfric=u(len(pv)), prest=u(len(pv)), overts=ov, oref=centroid(ov) if len(ov) else np.zeros((0, 2)),
                ofric=u(len(ov)), orest=u(len(ov)))


def stack(scenes):
    return {k: np.stack([s[k] for s in scenes]) for k in KEYS}


def rounded(batch, dtype):
    """the batch as the kernel reads it in dtype (float32: every value rounded to float32), as float64"""
    if dtype == torch.float64:
        return batch
    return {k: v.astype(np.float32).astype(np.float64) for k, v in batch.items()}


def box(x0, y0, x1, y1, nv=4):
    """axis-aligned box [x0, x1] x [y0, y1], positive area, padded to nv by repeating its last vertex"""
    v = [[x0, y0], [x1, y0], [x1, y1], [x0, y1]]
    return np.array(v + [v[-1]] * (nv - 4), np.float64)


def pad_at(V, nv, where):
    """polygon V [k, 2] padded to nv vertices by repeating its first ('first'), last ('last') or a middle vertex"""
    k = V.shape[0]
    at = {"first": 0, "last": k - 1, "middle": k // 2}[where]
    return np.concatenate([V[:at + 1], np.repeat(V[at:at + 1], nv - k, 0), V[at + 1:]])


def regular(n, cx, cy, r, a0):
    """regular n-gon of positive area, vertex k at angle a0 + 2 pi k / n"""
    k = np.arange(n)
    return np.stack([cx + r * np.cos(a0 + 2 * np.pi * k / n), cy + r * np.sin(a0 + 2 * np.pi * k / n)], 1)


def all_contact_scene(nb, no, nv=4, seed=0):
    """circles in a disc of radius 1 with radii 10 (every circle pair overlaps) and `no` obstacles that contain every
    circle centre (alternating orientation): every pair of the walk is a contact"""
    g = np.random.default_rng(seed)
    ang, rr = 2 * np.pi * g.random(nb), np.sqrt(g.random(nb))
    pos = np.stack([rr * np.cos(ang), rr * np.sin(ang)], 1)
    obs = []
    for k in range(no):
        b = box(-2.0 - k % 3, -2.0 - k % 5, 2.0 + k % 7, 2.0 + k % 2, nv)
        obs.append(b if k % 2 == 0 else np.concatenate([b[:4][::-1], b[4:]]))
    return make_scene(pos, 10.0, None, np.array(obs).reshape(no, nv, 2), nv, seed)


def random_scene(seed, nb, npoly, no, spread, nv=6):
    """circles, boxes (rotated, nearly axis-aligned and corner-on) and obstacles scattered over [0, spread]^2"""
    g = np.random.default_rng(seed)
    pos = spread * g.random((nb, 2))
    rad = 4 + 6 * g.random(nb)
    polys = []
    for k in range(npoly):
        x, y = spread * g.random(2)
        a = [2 * np.pi * g.random(), 1e-3 * (1 + g.random()), np.pi / 4 + 0.01 * (g.random() - 0.5)][k % 3]
        w, h = 10 + 20 * g.random(), 6 + 14 * g.random()
        polys.append(_rot_box(x, y, w, h, a, nv))
    obs = []
    for k in range(no):
        o = _rot_box(spread * g.random(), spread * g.random(), 30 + 40 * g.random(), 8 + 8 * g.random(),
                     0.5 * (g.random() - 0.5), nv)
        obs.append(o if k % 2 == 0 else np.concatenate([o[:4][::-1], o[4:]]))
    return make_scene(pos, rad, np.array(polys).reshape(npoly, nv, 2), np.array(obs).reshape(no, nv, 2), nv, seed)


def _rot_box(cx, cy, w, h, a, nv):
    c, s = math.cos(a), math.sin(a)
    loc = [(w / 2, -h / 2), (w / 2, h / 2), (-w / 2, h / 2), (-w / 2, -h / 2)]
    v = [[cx + c * x - s * y, cy + s * x + c * y] for x, y in loc]
    return np.array(v + [v[-1]] * (nv - 4))


def aligned_stack(nv=4):
    """integer-coordinate axis-aligned boxes, exact ties everywhere: a floor obstacle, boxes resting on it (touching
    and 1/4 deep), side by side (touching), equal boxes stacked, a wall, and circles resting on a box and on the
    floor"""
    floor = box(-40, 0, 40, 4, nv)
    wall = box(-44, -40, -40, 4, nv)[::-1] if nv == 4 else np.concatenate([box(-44, -40, -40, 4)[::-1],
                                                                           np.repeat(box(-44, -40, -40, 4)[:1], nv - 4, 0)])
    polys = [box(-30, -8, -22, 0, nv), box(-22, -8, -14, 0, nv),          # side by side, on the floor
             box(-30, -16, -22, -8, nv), box(-30, -24, -22, -16, nv),     # equal boxes stacked
             box(0, -6, 10, 0.25, nv), box(-40, -4, -36, 0, nv),          # 1/4 deep; in the floor-wall corner
             box(12, -4, 16, 0, nv), box(16, -4, 20, 0, nv),              # equal, touching, on the floor
             box(51.75, 1.75, 56, 6, nv),                                 # a box into a triangle's hypotenuse:
             np.array([[50, 0], [54, 0]] + [[50, 4]] * (nv - 2), np.float64)]   # body2 holds the reference face
    circles = [[-26.0, -25.0], [20.5, -1.0]]
    return make_scene(circles, 1.0, np.array(polys), np.array([floor, wall]), nv, seed=3)


def gon_scene():
    """regular 256-gons against boxes and against each other, posed so that the features name edges >= 128 and edge
    255: a 256-gon whose edge 255 faces down rests 0.05 deep on a slightly tilted box; a second one, a quarter step
    off its flat pose, rests on the first; a box leans its corner into the first one's left side"""
    n, r = 256, 20.0
    step = 2 * np.pi / n
    rin = r * np.cos(np.pi / n)
    g1 = regular(n, 0.0, 0.0, r, -np.pi / 2 - step * 255.5)                 # edge 255's normal points down (-y)
    g2 = regular(n, 0.0, 2 * rin - 0.05, r, -np.pi / 2 - step * 130.25)     # edge 130 nearly faces down
    lean = _rot_box(-rin - 3 * np.sqrt(2) + 0.03, 0.0, 6.0, 6.0, np.pi / 4 + 0.003, n)   # a corner 0.03 deep, left
    floor = _rot_box(0.0, -rin + 0.05 - 3.0, 30.0, 6.0, 0.002, n)
    return make_scene(None, None, np.stack([g1, g2, lean]), floor[None], n, seed=5)


def boundary_scenes(dtype):
    """scenes exactly on each rule's inclusive boundary (eps = 1/8) and one ulp (of dtype) past it, coordinates exact
    in float32: dict name -> (scene, expected count). Circle-circle: pen = -eps; circle-polygon: |c - q| - r = eps;
    hull-hull SAT: separation = eps (both ways, a tie); hull-hull clipped point: one point at distance eps; a circle
    centre on an edge and on a vertex."""
    f = np.float32 if dtype == torch.float32 else np.float64
    up = lambda x: float(np.nextafter(f(x), f(np.inf)))
    dn = lambda x: float(np.nextafter(f(x), f(-np.inf)))
    sq = box(0, 0, 4, 4)
    out = {}
    out["cc_at"] = (make_scene([[0, 0], [2.125, 0]], 1.0), 1)
    out["cc_past"] = (make_scene([[0, 0], [up(2.125), 0]], 1.0), 0)
    out["cp_at"] = (make_scene([[-1.125, 2]], 1.0, None, [sq]), 1)
    out["cp_past"] = (make_scene([[dn(-1.125), 2]], 1.0, None, [sq]), 0)
    out["cp_on_edge"] = (make_scene([[4, 2]], 1.0, None, [sq]), 1)
    out["cp_on_vertex"] = (make_scene([[4, 4]], 1.0, None, [sq]), 1)
    out["sat_at"] = (make_scene(None, None, [sq, box(4.125, 0, 8.125, 4)]), 2)
    out["sat_past"] = (make_scene(None, None, [sq, box(up(4.125), 0, 8.125, 4)]), 0)
    quad = lambda x: np.array([[4.0625, 0], [8, 0], [8, 4], [x, 4]])
    out["clip_at"] = (make_scene(None, None, [sq, quad(4.125)]), 2)
    out["clip_past"] = (make_scene(None, None, [sq, quad(up(4.125))]), 1)
    return out
