"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference's `World.step_dt` for circles, DYNAMIC convex polygons
(`Rect` / `Hull`, bodies.py:154-301) and static polygon obstacles (pinned `Rect` / `Hull`), in the reference's
formulation: bodies [circles..., polygons..., obstacles...], every obstacle pinned by a `TotalConstraint`.

Extends `oracle.obstacle_oracle.OracleObstacleWorld` with
  * the polygon bodies' vertices held as the reference holds `Hull.verts`: about the centroid, rotated by the CHANGE
    of p[0] at every `set_p` (bodies.py:202-214; `Rect` rotates v0, v1 and negates them, :278-283), including the
    reset to the start of the step when dt is halved (world.py:101-107);
  * the hull-hull rule of contacts.py:145-292 written as the reference's loops (test_separations, get_support,
    get_incident_edge, clip_segment_to_line), with one divergence: every SAT scan starts at edge 0 instead of the
    body's `last_sat_idx` (bodies.py:175, contacts.py:119-131, :149-153), which changes the result only on an exact
    tie between edge separations. `margins` records, for every hull-hull pair with contacts, how far the winning
    separation of the reference body's scan is from its runner-up and how far the two bodies' separations are from
    each other, so a test can assert that no recorded scene sits on such a tie;
  * circle-polygon contacts against moving polygons (the circle-hull rule of obstacle_oracle.circle_polygon).
PARITY PIN: tests/test_polygon_oracle.py against trajectories recorded from the unmodified reference
(tests/golden/bworld_polygons.npz).
"""
import torch

from .obstacle_oracle import OracleObstacleWorld, circle_polygon
from .world_oracle import OracleCircleWorld


def left_orthogonal(v):
    """utils.py:99-102."""
    return torch.stack([v[1], -v[0]])


def rotation_matrix(ang):
    """utils.py:105-112."""
    s, c = torch.sin(ang), torch.cos(ang)
    rot_mat = ang.new_empty(2, 2)
    rot_mat[0, 0] = rot_mat[1, 1] = c
    rot_mat[0, 1], rot_mat[1, 0] = -s, s
    return rot_mat


def get_support(points, direction):
    """contacts.py:207-217 (`>=`: the last maximal point wins)."""
    best_idx, best_norm = None, -1.0
    for i, p in enumerate(points):
        cur_norm = p.dot(direction).item()
        if cur_norm >= best_norm:
            best_idx, best_norm = i, cur_norm
    return points[best_idx], best_idx


def _edge_ok(verts, i):
    return (verts[(i + 1) % len(verts)] - verts[i]).norm().item() > 0


def _orient(verts):
    """1 for the orientation every reference Hull has (positive shoelace area: left_orthogonal(edge) is the outward
    normal), -1 for an obstacle given the other way round (its outward normal is then -left_orthogonal(edge))"""
    n = len(verts)
    area = sum((verts[i][0] * verts[(i + 1) % n][1] - verts[i][1] * verts[(i + 1) % n][0]).item() for i in range(n))
    return 1.0 if area > 0 else -1.0


def separations(verts1, pos1, verts2, pos2, eps):
    """test_separations, contacts.py:219-250, scanning from edge 0 (zero-length edges skipped). Returns (dist, normal, support index,
    edge norm, edge index, margin of the winner over the runner-up)."""
    n = len(verts1)
    o = _orient(verts1)
    best_dist, best = -1e10, None
    dists = []
    for idx in range(n):
        if not _edge_ok(verts1, idx):
            continue
        edge = verts1[(idx + 1) % n] - verts1[idx]
        edge_norm = edge.norm()
        normal = o * left_orthogonal(edge) / edge_norm
        support_point, support_idx = get_support(verts2, -normal)
        support_point = support_point + pos2 - pos1                     # adjust to hull1's frame
        dist = normal.dot(support_point - verts1[idx])
        dists.append(dist.item())
        if dist.item() > best_dist:
            if dist.item() > eps:
                return dist.item(), None, None, None, idx, None          # separating axis
            best_dist = dist.item()
            best = (dist, normal, support_idx, edge_norm, idx)
    dists.sort()
    margin = dists[-1] - dists[-2] if len(dists) > 1 else float("inf")
    return best[0].item(), best[1], best[2], best[3], best[4], margin


def get_incident_edge(ref_normal, inc_verts, inc_vertex):
    """contacts.py:253-267; with zero-length edges skipped, the edges before and from the vertex."""
    n = len(inc_verts)
    o = _orient(inc_verts)
    prev = next(e for e in ((inc_vertex - k) % n for k in range(1, n + 1)) if _edge_ok(inc_verts, e))
    nxt = next(e for e in ((inc_vertex + k) % n for k in range(n)) if _edge_ok(inc_verts, e))
    min_dot, best_edge = 1e10, -1
    for i in (prev, nxt):
        edge = inc_verts[(i + 1) % n] - inc_verts[i]
        inc_normal = o * left_orthogonal(edge) / edge.norm()
        dot = ref_normal.dot(inc_normal).item()
        if dot < min_dot:
            min_dot, best_edge = dot, i
    return best_edge


def clip_segment_to_line(verts, normal, offset):
    """contacts.py:270-292, quirks included (both endpoints behind the plane still give one interpolated point)."""
    clipped = []
    distance0 = normal.dot(verts[0]) + offset
    distance1 = normal.dot(verts[1]) + offset
    if distance0.item() >= 0.0:
        clipped.append(verts[0])
    if distance1.item() >= 0.0:
        clipped.append(verts[1])
    if distance0.item() * distance1.item() < 0.0 or len(clipped) < 2:
        interp = distance0 / (distance0 - distance1)
        clipped.append(verts[0] + interp * (verts[1] - verts[0]))
    return clipped


def hull_hull(v1, pos1, v2, pos2, eps, margins=None):
    """contacts.py:145-201 for hulls with vertices v1 / v2 about their centroids pos1 / pos2 (body1 = the lower
    index). Returns the contact list [(normal, p1, p2, penetration)]."""
    c1 = separations(v1, pos1, v2, pos2, eps)
    if c1[0] > eps:
        return []
    c2 = separations(v2, pos2, v1, pos1, eps)
    if c2[0] > eps:
        return []
    ref2 = c2[0] > c1[0]
    if ref2:
        _, normal, inc_vertex, edge_norm, ref_edge, margin = c2
        vr, pr, vi, pin = v2, pos2, v1, pos1
    else:
        _, normal, inc_vertex, edge_norm, ref_edge, margin = c1
        vr, pr, vi, pin = v1, pos1, v2, pos2
    half_edge_norm = edge_norm / 2
    inc_edge = get_incident_edge(normal, vi, inc_vertex)
    incident = [vi[inc_edge], vi[(inc_edge + 1) % len(vi)]]
    incident = [v + pin - pr for v in incident]
    clip_plane = left_orthogonal(normal)
    clipped = clip_segment_to_line(incident, clip_plane, half_edge_norm)
    if len(clipped) < 2:
        return []
    clipped = clip_segment_to_line(clipped, -clip_plane, half_edge_norm)
    pts = []
    for v in clipped:
        dist = normal.dot(v - vr[ref_edge])
        if dist.item() <= eps:
            pt1 = v + normal * -dist
            pt2 = pt1 + pr - pin
            pts.append((normal, pt2, pt1, -dist) if ref2 else (-normal, pt1, pt2, -dist))
    if pts and margins is not None:
        margins.append((margin, abs(c2[0] - c1[0])))
    return pts


class OracleHullWorld(OracleObstacleWorld):
    """Circles (pos [nc,2], rad, vel [nc,3], mass, restitution, fric_coeff) and polygon bodies given as the reference
    holds them, the dynamic ones first, then `n_static` pinned obstacles: `hull_verts` (list of [V, 2] vertices about
    the centroid at the initial pose, i.e. `Hull.verts`), `hull_p` [nh, 3] (rot, x, y), `hull_vel` [nh, 3],
    `hull_mass`, `hull_inertia` (the body's M[0, 0]), `hull_fric`, `hull_rest`, `hull_is_rect` (Rect's
    rotate_verts). A pinned obstacle is a Hull under a TotalConstraint, as in OracleObstacleWorld."""

    def __init__(self, pos, rad, vel, mass, restitution, fric_coeff, hull_verts, hull_p, hull_vel, hull_mass,
                 hull_inertia, hull_fric, hull_rest, hull_is_rect, n_static=0, gravity=100.0, dt=1.0 / 30, eps=0.1,
                 tol=1e-6, post_stab=False, max_iter=10):
        f64 = torch.float64
        t = lambda x: torch.as_tensor(x, dtype=f64)
        pos = t(pos).reshape(-1, 2)
        nc, nh = pos.shape[0], len(hull_verts)
        self.ncirc, self.no, self.npoly = nc, int(n_static), nh - int(n_static)
        self.ndyn = nc + self.npoly
        hull_p = t(hull_p).reshape(nh, 3)
        OracleCircleWorld.__init__(
            self, torch.cat([pos, hull_p[:, 1:]]), torch.cat([t(rad).reshape(-1), torch.ones(nh, dtype=f64)]),
            torch.cat([t(vel).reshape(nc, 3), t(hull_vel).reshape(nh, 3)]),
            torch.cat([t(mass).reshape(-1), t(hull_mass).reshape(-1)]),
            torch.cat([t(restitution).reshape(-1), t(hull_rest).reshape(-1)]),
            torch.cat([t(fric_coeff).reshape(-1), t(hull_fric).reshape(-1)]),
            gravity=gravity, static=list(range(self.ndyn, nc + nh)), dt=dt, eps=eps, tol=tol, post_stab=post_stab,
            max_iter=max_iter)
        hi = t(hull_inertia).reshape(-1)
        for k in range(nh):
            self.Md[3 * (nc + k)] = hi[k]
            self.p[nc + k, 0] = hull_p[k, 0]
        self.hverts = [t(v).clone() for v in hull_verts]              # Hull.verts, about the centroid
        self.is_rect = [bool(x) for x in hull_is_rect]
        self.held_rot = [self.p[nc + k, 0].clone() for k in range(nh)]
        self.margins = []
        self.find_contacts()

    def hull_world_verts(self, k):
        """World-frame vertices of polygon body ncirc + k."""
        return self.p[self.ncirc + k, 1:] + self.hverts[k]

    def _set_p(self, new_p):
        """World.set_p / Body.move: Hull.set_p rotates the held vertices by the change of p[0] (bodies.py:202-214)."""
        self.p = new_p
        for k in range(len(self.hverts)):
            b = self.ncirc + k
            rot = self.p[b, 0] - self.held_rot[k]
            if rot.item() != 0:
                rm = rotation_matrix(rot)
                vs = self.hverts[k]
                if self.is_rect[k]:                                   # Rect.rotate_verts (bodies.py:278-283)
                    vs[0] = rm.matmul(vs[0])
                    vs[1] = rm.matmul(vs[1])
                    vs[2] = -vs[0]
                    vs[3] = -vs[1]
                else:
                    for i in range(len(vs)):
                        vs[i] = rm.matmul(vs[i])
            self.held_rot[k] = self.p[b, 0].clone()

    def find_contacts(self):
        if not hasattr(self, "hverts"):
            self.contacts = []
            return
        cs = []
        nc, nd = self.ncirc, self.ndyn
        for i in range(nd):
            for j in range(i + 1, nd + self.no):
                if i < nc:
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
                    hit = circle_polygon(c, self.hull_world_verts(j - nc))
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
                    continue
                v1, v2 = list(self.hverts[i - nc]), list(self.hverts[j - nc])
                for nrm, p1, p2, pen in hull_hull(v1, self.p[i, 1:], v2, self.p[j, 1:], self.eps, self.margins):
                    cs.append((nrm, p1, p2, pen, i, j))
        self.contacts = cs

    def step(self):
        """world.py:83-122, with the positions set as World.set_p / Body.move set them."""
        dt = self.dt
        start_p = self.p.clone()
        self.v = self.solve_dynamics(dt)
        while True:
            self._set_p(start_p + self.v.reshape(self.nb, 3) * dt)
            self.find_contacts()
            if all(c[3].item() <= self.tol for c in self.contacts):
                break
            dt /= 2
            self._set_p(start_p.clone())
        if self.post_stab:
            dp = self.post_stabilization() / 2
            self._set_p(self.p + dp.reshape(self.nb, 3) * dt)
            self.find_contacts()
        self.t += dt

