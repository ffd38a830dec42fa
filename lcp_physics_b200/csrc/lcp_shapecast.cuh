// lcp_shapecast.cuh -- batched shape casts and translational sweeps against the bodies of BatchedWorld scenes
// (lcpb200_shapecast).
//
// Every case reduces to one cast primitive: a ray from a point x along a unit direction u' = s u (s = +-1) against a
// target feature inflated by a radius rho >= 0, hitting at the first entry into the Minkowski sum of the target and a
// disk of radius rho:
//   circle (c, R):     the ray against the circle (c, R + rho), raycast_kernel's formula: w = x - c, b = u' . w,
//                      k = |w|^2 - (R + rho)^2; a miss if k < 0 (overlapping at t = 0), b >= 0 or b^2 - k < 0, else
//                      t = k / (-b + sqrt(b^2 - k)); normal m = (w + t u') / (R + rho); target feat 0.
//   polygon face e:    (edges of non-zero length, edge_ok) the offset line n_e . (y - v_e) = rho: den = n_e . u' < 0,
//                      t = (n_e . (v_e - x) + rho) / den >= 0, and the hit point within the offset edge; m = n_e,
//                      target feat e. The edge test is the projection of the hit point onto the edge lying in [0, 1],
//                      evaluated as the signs of u' x (a - x) at the offset edge's endpoints a: the endpoint values of
//                      the unoffset vertices are computed once per vertex and shared by the two edges that meet there,
//                      so that at rho = 0 a ray through a vertex cannot slip between two faces by round-off.
//   polygon vertex v:  (rho > 0 only) the circle (v, rho) with the circle rule; m = (w + t u') / rho, target feat
//                      256 + v.
// Within a polygon the faces come first, then the vertices, each in index order, and only a strictly nearer hit
// replaces the best. A target the swept shape already overlaps at t = 0 is skipped (the raycast convention carried
// over to shapes); one it only touches gives t = 0 when the motion heads into it and no hit otherwise.
//
// Disk mode (body_q == nullptr): query k sweeps a disk of radius r from origin o along u against every active body of
// its scene: x = o, s = +1, rho = r; a polygon is skipped when its signed distance at o (point_polygon) is < r.
// Body mode: query k translates body q = body_q[k] along u by at most limit[k] against every other active body not
// excluded by no_contact, held still:
//   circle q - circle j:      x = c_q, s = +1, the circle j with rho = R_q;
//   circle q - polygon j:     x = c_q, s = +1, polygon j with rho = R_q (skipped when sdf(c_q, j) < R_q);
//   polygon q - circle j:     x = c_j, s = -1, polygon q with rho = R_j (skipped when sdf(c_j, q) < R_j): the mover is
//                             the target;
//   polygon q - polygon j:    every vertex of q with s = +1 against j, then every vertex of j with s = -1 against q,
//                             rho = 0, the first strictly nearest wins; skipped when both cts::separation values are
//                             < 0 (overlapping).
// Bodies are visited in index order: from best = limit (max_dist in disk mode), body -1, a body replaces the best iff
// (body < 0 ? t <= best : t < best). feat packs the choices as dist_feat does: bits 0-8 the target feature, bits 9-16
// the source vertex (0 for a circle source), bit 17 set iff the source is the hit body (the mover is the target).
// Outputs: dist = t; normal = m in disk mode, and in body mode the unit normal from the mover towards the hit body
// (-m, or m when the mover is the target); point = x + s t u - R_src m, plus t u when the mover is the target (R_src:
// the source circle's radius, 0 for a vertex), the contact point at the time of impact. A miss (also a zero or
// non-finite direction, a non-finite origin or limit, a negative or non-finite radius, an inactive or out-of-range
// mover) reads dist = the limit, body -1, feat -1, zero normal and point.
//
// Layout: that of distance_kernel, one CTA per (scene, chunk of blockDim.x queries) work item, one query per thread,
// the best hit in registers. A body mover is read from global memory (load_body); the candidates are staged through
// shared memory by SceneWalk and read through LoadedEdges, as in nearest mode. No atomics; the result depends neither
// on the chunking nor on the tile sizes.
#pragma once
#include "lcp_distance.cuh"

namespace lcpb200 {
namespace ray {

// A cast's result and the choices behind it
template <typename T>
struct Cast {
  T t;                    // +inf: no hit
  T x, y, r;              // the source point and its radius R_src
  T mx, my;               // the target's normal m at the hit
  int feat;               // dist_feat
};

// the ray x + t u (w = x - c) against the circle of radius rr: raycast_kernel's entry rule
template <typename T>
__device__ __forceinline__ bool cast_circle(T wx, T wy, T ux, T uy, T rr, T& t) {
  const T b = ux * wx + uy * wy;
  const T k = wx * wx + wy * wy - rr * rr;
  if (k < T(0) || b >= T(0)) return false;
  const T disc = b * b - k;
  if (disc < T(0)) return false;
  t = k / (-b + sqrt(disc));
  return true;
}

// the ray x + t u (t >= 0) against the polygon g inflated by rho (faces, then vertex disks when rho > 0): t (+inf: no
// hit), the target feat and the normal m
template <typename T, class G>
__device__ __forceinline__ void cast_polygon(const G& g, int nv, T xx, T xy, T ux, T uy, T rho, T& t, int& tf, T& mx,
                                             T& my) {
  const T* P = g.P;
  t = T(INFINITY); tf = 0; mx = my = T(0);
  auto side = [&](int v) { return ux * (P[2 * v + 1] - xy) - uy * (P[2 * v] - xx); };
  const T c0 = side(0);
  T ce = c0;
  for (int e = 0; e < nv; ++e) {
    const int f = e + 1 == nv ? 0 : e + 1;
    const T cf = f == 0 ? c0 : side(f);
    if (g.ok(e)) {
      const T nx = g.nx(e), ny = g.ny(e);
      const T den = nx * ux + ny * uy;
      if (den < T(0)) {
        const T te = (nx * (P[2 * e] - xx) + ny * (P[2 * e + 1] - xy) + rho) / den;
        const T un = rho * (ux * ny - uy * nx);          // u x (rho n_e): the offset edge's endpoints
        const T ca = ce + un, cb = cf + un;
        const bool within = !(ca > T(0) && cb > T(0)) && !(ca < T(0) && cb < T(0));
        if (te >= T(0) && within && te < t) { t = te; tf = e; mx = nx; my = ny; }
      }
    }
    ce = cf;
  }
  if (rho > T(0)) {
    for (int v = 0; v < nv; ++v) {
      const T wx = xx - P[2 * v], wy = xy - P[2 * v + 1];
      T tv;
      if (cast_circle(wx, wy, ux, uy, rho, tv) && tv < t) {
        t = tv; tf = 256 + v;
        mx = (wx + tv * ux) / rho; my = (wy + tv * uy) / rho;
      }
    }
  }
}

// A (the mover, or the swept disk) translated along u against C, held still: the rule above
template <typename T, class G>
__device__ __forceinline__ Cast<T> sweep_pair(const Side<T, G>& A, const Side<T, G>& C, int nv, T ux, T uy) {
  Cast<T> c;
  c.t = T(INFINITY); c.x = c.y = c.r = c.mx = c.my = T(0); c.feat = 0;
  if (A.circle || C.circle) {
    const bool src_b = !A.circle;                        // a circle is the source, the mover first
    const T x = src_b ? C.cx : A.cx, y = src_b ? C.cy : A.cy, rho = src_b ? C.r : A.r;
    const T sx = src_b ? -ux : ux, sy = src_b ? -uy : uy;
    int tf = 0;
    if (A.circle && C.circle) {
      const T wx = x - C.cx, wy = y - C.cy, rr = C.r + rho;
      T t;
      if (!cast_circle(wx, wy, sx, sy, rr, t)) return c;
      c.t = t; c.mx = (wx + t * sx) / rr; c.my = (wy + t * sy) / rr;
    } else {
      const G g = src_b ? A.g : C.g;                     // the polygon is the target
      T smax, dmin, qdx, qdy;
      int emax, emin;
      point_polygon(g, nv, x, y, smax, emax, dmin, emin, qdx, qdy);
      if (emax < 0 || (smax <= T(0) ? smax : sqrt(dmin)) < rho) return c;   // no edge, or overlapping at t = 0
      cast_polygon(g, nv, x, y, sx, sy, rho, c.t, tf, c.mx, c.my);
    }
    c.x = x; c.y = y; c.r = rho;
    c.feat = dist_feat(tf, 0, src_b);
    return c;
  }
  const cts::Sep<T> sa = cts::separation(A.g.P, A.o, C.g.P, nv);
  const cts::Sep<T> sb = cts::separation(C.g.P, C.o, A.g.P, nv);
  if (!(sa.dist >= T(0) || sb.dist >= T(0))) return c;  // overlapping, no edge or a non-finite vertex
  for (int src_b = 0; src_b < 2; ++src_b) {              // A's vertices along u, then C's along -u
    const G S = src_b ? C.g : A.g, Tg = src_b ? A.g : C.g;
    const T sx = src_b ? -ux : ux, sy = src_b ? -uy : uy;
    for (int i = 0; i < nv; ++i) {
      const T vx = S.P[2 * i], vy = S.P[2 * i + 1];
      T t, mx, my;
      int tf;
      cast_polygon(Tg, nv, vx, vy, sx, sy, T(0), t, tf, mx, my);
      if (t < c.t) {
        c.t = t; c.x = vx; c.y = vy; c.mx = mx; c.my = my;
        c.feat = dist_feat(tf, i, src_b);
      }
    }
  }
  return c;
}

template <typename T>
__global__ void __launch_bounds__(NT) shapecast_kernel(CastArgs<T> a, int chunks) {
  const SceneWalk<T> walk(a.bd);
  const cts::Bodies<T>& bd = a.bd;
  const int tid = walk.tid, nth = walk.nth, nv = walk.nv, nt = walk.nt;
  const bool disk = a.body_q == nullptr;
  const long long items = (long long)a.B * chunks;
  for (long long it = blockIdx.x; it < items; it += gridDim.x) {
    const int sc = (int)(it / chunks);
    const int r = (int)(it - (long long)sc * chunks) * nth + tid;
    const bool live = r < a.K;
    const size_t ri = (size_t)sc * a.K + (live ? r : 0);
    const uint32_t* aw = a.active ? a.active + (size_t)sc * walk.words : nullptr;
    auto on = [&](int b) { return b >= 0 && b < nt && (!aw || ((__ldg(aw + (b >> 5)) >> (b & 31)) & 1u)); };
    T ux = T(0), uy = T(0), lim = disk ? a.max_dist : T(0);
    if (live) {
      ux = a.dir[2 * ri]; uy = a.dir[2 * ri + 1];
      if (!disk) lim = a.limit[ri];
    }
    bool valid = live && isfinite(ux) && isfinite(uy) && ux * ux + uy * uy > T(0) && isfinite(lim) && lim >= T(0);
    const int iq = live && !disk ? a.body_q[ri] : -1;
    Side<T, LoadedEdges<T>> A;
    if (disk) {
      T ox = T(0), oy = T(0), rr = T(0);
      if (live) { ox = a.origin[2 * ri]; oy = a.origin[2 * ri + 1]; rr = a.radius[ri]; }
      valid = valid && isfinite(ox) && isfinite(oy) && isfinite(rr) && rr >= T(0);
      A = Side<T, LoadedEdges<T>>{true, ox, oy, rr, LoadedEdges<T>{nullptr, T(0), nv}, T(0)};
    } else {
      valid = valid && on(iq);
      A = load_body(bd, sc, valid ? iq : 0);
    }
    T best = lim;
    int bbody = -1;
    Cast<T> bc;
    bc.x = bc.y = bc.r = bc.mx = bc.my = T(0); bc.feat = -1;
    const uint32_t* nc = !disk && a.no_contact ? a.no_contact + (size_t)sc * a.nc_stride : nullptr;
    auto excluded = [&](int j) {
      if (!nc) return false;
      const long long bit = (long long)(iq < j ? iq : j) * nt + (iq < j ? j : iq);
      return ((__ldg(nc + (bit >> 5)) >> (bit & 31)) & 1u) != 0u;
    };
    auto visit = [&](int j, const Side<T, LoadedEdges<T>>& C) {
      const Cast<T> c = sweep_pair(A, C, nv, ux, uy);
      if (bbody < 0 ? c.t <= best : c.t < best) { best = c.t; bbody = j; bc = c; }
    };
    walk(sc, aw, valid,
      [&](int j, T cx, T cy, T cr) {
        if (j == iq || excluded(j)) return;
        visit(j, Side<T, LoadedEdges<T>>{true, cx, cy, cr, LoadedEdges<T>{nullptr, T(0), nv}, T(0)});
      },
      [&](int j, const T* P, const T*, const unsigned char*, int o) {
        if (j == iq || excluded(j)) return;
        visit(j, Side<T, LoadedEdges<T>>{false, T(0), T(0), T(0), LoadedEdges<T>{P, T(o), nv}, T(o)});
      });
    if (live) {
      const bool hit = bbody >= 0;
      const bool src_b = hit && ((bc.feat >> 17) & 1);
      const T sg = disk || src_b ? T(1) : T(-1);
      const T tu = src_b ? T(0) : best;                  // the mover as the target: its t u cancels s t u
      a.dist[ri] = best;
      a.body[ri] = bbody;
      a.feat[ri] = hit ? bc.feat : -1;
      a.normal[2 * ri] = hit ? sg * bc.mx : T(0);
      a.normal[2 * ri + 1] = hit ? sg * bc.my : T(0);
      a.point[2 * ri] = hit ? bc.x + tu * ux - bc.r * bc.mx : T(0);
      a.point[2 * ri + 1] = hit ? bc.y + tu * uy - bc.r * bc.my : T(0);
    }
  }
}

}  // namespace ray
}  // namespace lcpb200
