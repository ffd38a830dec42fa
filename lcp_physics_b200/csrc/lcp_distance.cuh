// lcp_distance.cuh -- batched distances between the bodies of BatchedWorld scenes (lcpb200_body_distance).
//
// Every pair (A, B) reduces to the signed distance of one feature point of one body (the source: a circle's centre
// with its radius r, or a polygon's vertex with r = 0) to the other body (the target), minus r, with the target-side
// choices of sdf_kernel (lcp_sdf.cuh):
//   circle i - circle j:       source the centre of i, d = |c_i - c_j| - r_j - r_i, target feat circle.
//   circle - polygon:          source the circle's centre (either order), d = sdf(centre, polygon) - r, sdf's feat.
//   polygon - polygon:         S = max over the faces of both polygons of min over the other's vertices of
//                              n_e . (v - v_e) (cts::separation both ways; A's faces win a tie).
//     separated (S > 0):       the exact Euclidean distance: min over A's vertices of their outside distance to B and
//                              over B's vertices of theirs to A (compared squared; the first vertex wins a tie, A's
//                              before B's); target feat e, the nearest edge.
//     overlapping (S <= 0):    d = S, the minimum translation distance; source the support vertex of the SAT axis
//                              (separation's: the last maximal vertex), target feat 256 + e of the SAT face.
// n is the unit normal from A towards B (moving B along n increases d): minus the target's sdf normal m when A is
// the source, m when B is. point_a, the witness on A, is source - r m (A the source) or source - sdf m (B the source),
// so that point_b = point_a + d n is the other witness; zero m (a source on the target's closest point) gives zero n.
// Pair mode reads (body_a, body_b) per query; nearest mode reads body_a and takes the nearest other active body not
// excluded by no_contact, visited in index order: starting from best = max_dist, body -1, a body replaces the best iff
// (body < 0 ? d <= best : d < best). A query whose body is inactive, out of range or named twice, or with nothing
// within max_dist, reads dist = max_dist, body -1, feat -1 and zero normal and point_a.
//
// Layout: that of sdf_kernel, one CTA per (scene, chunk of blockDim.x queries) work item, one query per thread. The
// query's own body (both bodies in pair mode) is read from global memory; in nearest mode the candidates are staged
// through shared memory by SceneWalk (lcp_raycast.cuh). A staged candidate is read through the same edge view as a
// body read from global memory (LoadedEdges over its staged vertices: the same expressions for edge flags and
// normals), so that both modes run the same source expressions. No atomics.
#pragma once
#include "lcp_sdf.cuh"

namespace lcpb200 {
namespace ray {

// feat of a body distance: bits 0-8 the target's sdf feat (e or 256 + e; 0 for a circle target), bits 9-16 the
// source vertex (0 for a circle source), bit 17 set iff B is the source
__host__ __device__ __forceinline__ int dist_feat(int tfeat, int vtx, int src_b) { return tfeat | vtx << 9 | src_b << 17; }

// One body of a pair: a circle (centre cx, cy, radius r), or a polygon of edge view g and orientation o (+-1)
template <typename T, class G>
struct Side {
  bool circle;
  T cx, cy, r;
  G g;
  T o;
};

// A pair's distance and the choices behind it
template <typename T>
struct Pair {
  T d;                    // the distance (+inf: a polygon without an edge of non-zero length, never a hit)
  T x, y;                 // the source point
  T w;                    // point_a = source - w m: r (A the source) or the source's sdf (B the source)
  T mx, my, mlen;         // the target's sdf normal at the source, m = (mx, my) / mlen (mlen == 0: zero)
  int feat;               // dist_feat
};

// sdf of (px, py) to body b (the rule of sdf_kernel): s, the unnormalised normal (mx, my) / mlen and the feat;
// false for a polygon without an edge of non-zero length
template <typename T, class G>
__device__ __forceinline__ bool point_body(const Side<T, G>& b, int nv, T px, T py, T& s, T& mx, T& my, T& mlen,
                                           int& tf) {
  if (b.circle) {
    const T dx = px - b.cx, dy = py - b.cy;
    const T d = sqrt(dx * dx + dy * dy);
    s = d - b.r; mx = dx; my = dy; mlen = d; tf = 0;
    return true;
  }
  T smax, dmin, qdx, qdy;
  int emax, emin;
  point_polygon(b.g, nv, px, py, smax, emax, dmin, emin, qdx, qdy);
  if (emax < 0) return false;
  if (smax <= T(0)) { s = smax; mx = b.g.nx(emax); my = b.g.ny(emax); mlen = T(1); tf = 256 + emax; }
  else { s = sqrt(dmin); mx = qdx; my = qdy; mlen = s; tf = emin; }
  return true;
}

// the nearest vertex of polygon S to polygon G (outside distances, squared): replaces (best, ...) iff strictly nearer
template <typename T, class GS, class GT>
__device__ __forceinline__ void nearest_vertex(const GS& S, const GT& G, int nv, int src_b, T& best, Pair<T>& p) {
  for (int i = 0; i < nv; ++i) {
    const T vx = S.P[2 * i], vy = S.P[2 * i + 1];
    T smax, dmin, qdx, qdy;
    int emax, emin;
    point_polygon(G, nv, vx, vy, smax, emax, dmin, emin, qdx, qdy);
    if (dmin < best) {
      best = dmin;
      p.x = vx; p.y = vy; p.mx = qdx; p.my = qdy;
      p.feat = dist_feat(emin, i, src_b);
    }
  }
}

template <typename T, class GA, class GB>
__device__ __forceinline__ Pair<T> pair_distance(const Side<T, GA>& A, const Side<T, GB>& B, int nv) {
  Pair<T> p;
  p.d = T(INFINITY); p.x = p.y = p.w = p.mx = p.my = p.mlen = T(0); p.feat = 0;
  T s;
  int tf;
  if (A.circle || B.circle) {
    const bool src_b = !A.circle;                        // a circle's centre is the source, A's first
    const T x = src_b ? B.cx : A.cx, y = src_b ? B.cy : A.cy, r = src_b ? B.r : A.r;
    const bool ok = src_b ? point_body(A, nv, x, y, s, p.mx, p.my, p.mlen, tf)
                          : point_body(B, nv, x, y, s, p.mx, p.my, p.mlen, tf);
    if (!ok) return p;
    p.d = s - r; p.x = x; p.y = y; p.w = src_b ? s : r;
    p.feat = dist_feat(tf, 0, src_b);
    return p;
  }
  const cts::Sep<T> sa = cts::separation(A.g.P, A.o, B.g.P, nv);     // A's faces, support vertices of B
  const cts::Sep<T> sb = cts::separation(B.g.P, B.o, A.g.P, nv);     // B's faces, support vertices of A
  if (!(sa.dist > T(-INFINITY) && sb.dist > T(-INFINITY))) return p;  // no edge, or a non-finite vertex
  if (!(sa.dist > T(0) || sb.dist > T(0))) {
    if (sb.dist > sa.dist) {                             // B's face e, source A's support vertex
      p.d = sb.dist; p.x = A.g.P[2 * sb.sup]; p.y = A.g.P[2 * sb.sup + 1]; p.w = T(0);
      p.mx = B.g.nx(sb.edge); p.my = B.g.ny(sb.edge); p.mlen = T(1);
      p.feat = dist_feat(256 + sb.edge, sb.sup, 0);
    } else {                                             // A's face e, source B's support vertex
      p.d = sa.dist; p.x = B.g.P[2 * sa.sup]; p.y = B.g.P[2 * sa.sup + 1]; p.w = sa.dist;
      p.mx = A.g.nx(sa.edge); p.my = A.g.ny(sa.edge); p.mlen = T(1);
      p.feat = dist_feat(256 + sa.edge, sa.sup, 1);
    }
    return p;
  }
  T best = T(INFINITY);
  nearest_vertex(A.g, B.g, nv, 0, best, p);
  nearest_vertex(B.g, A.g, nv, 1, best, p);
  p.d = sqrt(best); p.mlen = p.d;
  p.w = (p.feat >> 17) ? p.d : T(0);
  return p;
}

// body b of scene sc read from global memory
template <typename T>
__device__ __forceinline__ Side<T, LoadedEdges<T>> load_body(const cts::Bodies<T>& bd, int sc, int b) {
  Side<T, LoadedEdges<T>> s;
  s.circle = b < bd.nb;
  s.cx = s.cy = s.r = s.o = T(0);
  s.g = LoadedEdges<T>{nullptr, T(0), bd.nv};
  if (s.circle) {
    const size_t g = (size_t)sc * bd.nb + b;
    s.cx = bd.pos[2 * g]; s.cy = bd.pos[2 * g + 1]; s.r = bd.rad[g];
  } else {
    s.g.P = bd.verts(sc, b);
    s.o = s.g.o = cts::poly_orient(s.g.P, bd.nv);
  }
  return s;
}

template <typename T>
__global__ void __launch_bounds__(NT) distance_kernel(DistArgs<T> a, int chunks) {
  const SceneWalk<T> walk(a.bd);
  const cts::Bodies<T>& bd = a.bd;
  const int tid = walk.tid, nth = walk.nth, nv = walk.nv, nt = walk.nt;
  const bool nearest = a.body_b == nullptr;
  const T maxd = a.max_dist;
  const long long items = (long long)a.B * chunks;
  for (long long it = blockIdx.x; it < items; it += gridDim.x) {
    const int sc = (int)(it / chunks);
    const int r = (int)(it - (long long)sc * chunks) * nth + tid;
    const bool live = r < a.K;
    const size_t ri = (size_t)sc * a.K + (live ? r : 0);
    const size_t qi = a.shared_queries ? (size_t)(live ? r : 0) : ri;
    const uint32_t* aw = a.active ? a.active + (size_t)sc * walk.words : nullptr;
    auto on = [&](int b) { return b >= 0 && b < nt && (!aw || ((__ldg(aw + (b >> 5)) >> (b & 31)) & 1u)); };
    const int ia = live ? a.body_a[qi] : -1;
    const int ib = live && !nearest ? a.body_b[qi] : -1;
    const bool valid = live && on(ia) && (nearest || (ib != ia && on(ib)));
    Side<T, LoadedEdges<T>> A = load_body(bd, sc, valid ? ia : 0);
    T best = maxd;
    int bbody = -1;
    Pair<T> bp;
    bp.x = bp.y = bp.w = bp.mx = bp.my = bp.mlen = T(0); bp.feat = -1;
    if (!nearest) {
      if (valid) {
        const Pair<T> p = pair_distance(A, load_body(bd, sc, ib), nv);
        if (p.d <= best) { best = p.d; bbody = ib; bp = p; }
      }
    } else {
      const uint32_t* nc = a.no_contact ? a.no_contact + (size_t)sc * a.nc_stride : nullptr;
      auto excluded = [&](int j) {
        if (!nc) return false;
        const long long bit = (long long)(ia < j ? ia : j) * nt + (ia < j ? j : ia);
        return ((__ldg(nc + (bit >> 5)) >> (bit & 31)) & 1u) != 0u;
      };
      auto visit = [&](int j, const Side<T, LoadedEdges<T>>& C) {
        const Pair<T> p = pair_distance(A, C, nv);
        if (bbody < 0 ? p.d <= best : p.d < best) { best = p.d; bbody = j; bp = p; }
      };
      walk(sc, aw, valid,
        [&](int j, T cx, T cy, T cr) {
          if (j == ia || excluded(j)) return;
          visit(j, Side<T, LoadedEdges<T>>{true, cx, cy, cr, LoadedEdges<T>{nullptr, T(0), nv}, T(0)});
        },
        [&](int j, const T* P, const T*, const unsigned char*, int o) {
          if (j == ia || excluded(j)) return;
          visit(j, Side<T, LoadedEdges<T>>{false, T(0), T(0), T(0), LoadedEdges<T>{P, T(o), nv}, T(o)});
        });
    }
    if (live) {
      const bool hit = bbody >= 0;
      const T ux = bp.mlen > T(0) ? bp.mx / bp.mlen : T(0), uy = bp.mlen > T(0) ? bp.my / bp.mlen : T(0);
      const T sg = (bp.feat >> 17) & 1 ? T(1) : T(-1);
      a.dist[ri] = best;
      a.body[ri] = bbody;
      a.feat[ri] = hit ? bp.feat : -1;
      a.normal[2 * ri] = hit ? sg * ux : T(0);
      a.normal[2 * ri + 1] = hit ? sg * uy : T(0);
      a.point_a[2 * ri] = hit ? bp.x - bp.w * ux : T(0);
      a.point_a[2 * ri + 1] = hit ? bp.y - bp.w * uy : T(0);
    }
  }
}

}  // namespace ray
}  // namespace lcpb200
