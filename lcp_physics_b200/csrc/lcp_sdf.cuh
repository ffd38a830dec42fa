// lcp_sdf.cuh -- batched signed distances to the bodies of BatchedWorld scenes (lcpb200_signed_distance).
//
// A query point x is tested against the body list [circles, dynamic polygons, obstacles] of its scene, inactive bodies
// skipped:
//   circle (c, r):    sdf = |x - c| - r, feat -1, normal (x - c) / |x - c| ((0, 0) when x == c).
//   convex polygon:   either orientation (poly_orient), zero-length padding edges skipped (edge_ok). Edge e runs from
//                     v_e to v_f, E = v_f - v_e, outward unit normal n_e, s_e = n_e . (x - v_e).
//                     inside (every s_e <= 0): sdf = max_e s_e, feat 256 + e of the largest (the first on a tie),
//                     normal n_e.
//                     outside: t = clamp((x - v_e) . E / |E|^2, 0, 1), q_e = v_e if t <= 0, v_f (the loaded vertex)
//                     if t >= 1, else v_e + t E; sdf = min_e |x - q_e| (compared as |x - q_e|^2; the first edge wins a
//                     tie, so the two edges meeting at a vertex tie exactly in its region and the lower one is
//                     reported), feat e, normal (x - q) / |x - q|.
// The smallest sdf wins, an exact tie goes to the lower body index: starting from best = max_dist, body -1, a body
// replaces the best iff (body < 0 ? sdf <= best : sdf < best). Nothing within max_dist, or a non-finite point: body -1,
// feat -1, sdf = max_dist, normal (0, 0). This is the exact Euclidean signed distance of one circle or convex polygon;
// over overlapping bodies it is the min of their distances, exact outside every body and a bound inside.
//
// Layout: one CTA per (scene, chunk of blockDim.x points) work item, one point per thread, the best (sdf, body, feat,
// normal) in registers; the bodies are staged through shared memory by SceneWalk (lcp_raycast.cuh). Every thread
// visits the bodies in index order, so the result depends neither on the chunking nor on the tile sizes. No atomics.
#pragma once
#include "lcp_raycast.cuh"

namespace lcpb200 {
namespace ray {

// The edges of a polygon staged by SceneWalk: vertex e at P[2 e], edge flag ok[e] (edge_ok), outward unit normal
// N[2 e].
template <typename T>
struct StagedEdges {
  const T* P;
  const T* N;
  const unsigned char* ok_;
  __device__ __forceinline__ bool ok(int e) const { return ok_[e]; }
  __device__ __forceinline__ T nx(int e) const { return N[2 * e]; }
  __device__ __forceinline__ T ny(int e) const { return N[2 * e + 1]; }
};

// The vertices of a polygon moved rigidly on every read (time_of_impact, lcp_toi.cuh): stored vertex v maps to
// v + (R(phi) - I)(v - c) + s, with cm1 = cos(phi) - 1 and sn = sin(phi). At phi = 0 and s = 0 every read returns the
// stored value exactly.
template <typename T>
struct MovedVerts {
  const T* P;
  T cm1, sn, cx, cy, sx, sy;
  __device__ __forceinline__ T operator[](int i) const {
    const int v = i >> 1;
    const T wx = P[2 * v] - cx, wy = P[2 * v + 1] - cy;
    return (i & 1) ? P[i] + ((sn * wx + cm1 * wy) + sy) : P[i] + ((cm1 * wx - sn * wy) + sx);
  }
};

// The edges of a polygon whose normals were not staged (vertices P, orientation o from poly_orient): the flag and the
// normal computed with the expressions of SceneWalk. V: the vertex access, a pointer or MovedVerts.
template <typename T, class V = const T*>
struct LoadedEdges {
  V P;
  T o;
  int nv;
  __device__ __forceinline__ bool ok(int e) const { return cts::edge_ok(P, nv, e); }
  __device__ __forceinline__ T ex(int e) const { return P[2 * (e + 1 == nv ? 0 : e + 1)] - P[2 * e]; }
  __device__ __forceinline__ T ey(int e) const { return P[2 * (e + 1 == nv ? 0 : e + 1) + 1] - P[2 * e + 1]; }
  __device__ __forceinline__ T nx(int e) const {
    const T x = ex(e), y = ey(e);
    return o * y / sqrt(x * x + y * y);
  }
  __device__ __forceinline__ T ny(int e) const {
    const T x = ex(e), y = ey(e);
    return -o * x / sqrt(x * x + y * y);
  }
};

// The choices of the signed distance of point (px, py) to one convex polygon g (StagedEdges or LoadedEdges of nv
// vertices, read through g.P), the rule above: smax / emax the largest s_e and its edge (emax < 0: no edge of non-zero
// length), dmin / emin the smallest |x - q_e|^2 and its edge, (qdx, qdy) = x - q of that edge. Shared by sdf_kernel,
// distance_kernel (lcp_distance.cuh) and toi_kernel (lcp_toi.cuh).
template <typename T, class G>
__device__ __forceinline__ void point_polygon(const G& g, int nv, T px, T py, T& smax, int& emax, T& dmin, int& emin,
                                              T& qdx, T& qdy) {
  const auto& P = g.P;
  smax = T(-INFINITY); dmin = T(INFINITY); qdx = T(0); qdy = T(0);
  emax = -1; emin = -1;
  for (int e = 0; e < nv; ++e) {
    if (!g.ok(e)) continue;
    const int f = e + 1 == nv ? 0 : e + 1;
    const T vx = P[2 * e], vy = P[2 * e + 1];
    const T wx = px - vx, wy = py - vy;
    const T s = g.nx(e) * wx + g.ny(e) * wy;
    if (s > smax) { smax = s; emax = e; }
    const T ex = P[2 * f] - vx, ey = P[2 * f + 1] - vy;
    const T t = (wx * ex + wy * ey) / (ex * ex + ey * ey);
    T dx, dy;
    if (t <= T(0)) { dx = wx; dy = wy; }
    else if (t >= T(1)) { dx = px - P[2 * f]; dy = py - P[2 * f + 1]; }
    else { dx = px - (vx + t * ex); dy = py - (vy + t * ey); }
    const T d2 = dx * dx + dy * dy;
    if (d2 < dmin) { dmin = d2; emin = e; qdx = dx; qdy = dy; }
  }
}

template <typename T>
__global__ void __launch_bounds__(NT) sdf_kernel(SdfArgs<T> a, int chunks) {
  const SceneWalk<T> walk(a.bd);
  const int tid = walk.tid, nth = walk.nth, nv = walk.nv;
  const T maxd = a.max_dist;
  const long long items = (long long)a.B * chunks;
  for (long long it = blockIdx.x; it < items; it += gridDim.x) {
    const int sc = (int)(it / chunks);
    const int r = (int)(it - (long long)sc * chunks) * nth + tid;
    const bool live = r < a.Q;
    const size_t ri = (size_t)sc * a.Q + (live ? r : 0);
    const size_t pi = a.shared_points ? (size_t)(live ? r : 0) : ri;
    T px = T(0), py = T(0);
    if (live) { px = a.points[2 * pi]; py = a.points[2 * pi + 1]; }
    const bool valid = live && isfinite(px) && isfinite(py);
    const uint32_t* aw = a.active ? a.active + (size_t)sc * walk.words : nullptr;
    // the best body's normal is (bnx, bny) / blen: blen = |x - q| outside, 1 inside a polygon, 0 at a circle's centre
    T best = maxd, bnx = T(0), bny = T(0), blen = T(0);
    int bbody = -1, bfeat = -1;
    walk(sc, aw, valid,
      [&](int j, T cx, T cy, T cr) {
        const T dx = px - cx, dy = py - cy;
        const T d = sqrt(dx * dx + dy * dy);
        const T s = d - cr;
        if (bbody < 0 ? s <= best : s < best) {
          best = s; bbody = j; bfeat = -1;
          bnx = dx; bny = dy; blen = d;
        }
      },
      [&](int j, const T* P, const T* N, const unsigned char* ok, int) {
        T smax, dmin, qdx, qdy;
        int emax, emin;
        point_polygon(StagedEdges<T>{P, N, ok}, nv, px, py, smax, emax, dmin, emin, qdx, qdy);
        if (emax < 0) return;                            // no edge of non-zero length
        const bool inside = smax <= T(0);
        const T s = inside ? smax : sqrt(dmin);
        if (bbody < 0 ? s <= best : s < best) {
          best = s; bbody = j;
          if (inside) { bfeat = 256 + emax; bnx = N[2 * emax]; bny = N[2 * emax + 1]; blen = T(1); }
          else { bfeat = emin; bnx = qdx; bny = qdy; blen = s; }
        }
      });
    if (live) {
      a.sdf[ri] = best;
      a.body[ri] = bbody;
      a.feat[ri] = bfeat;
      if (a.normal) {
        const bool nz = blen > T(0);
        a.normal[2 * ri] = nz ? bnx / blen : T(0);
        a.normal[2 * ri + 1] = nz ? bny / blen : T(0);
      }
    }
  }
}

}  // namespace ray
}  // namespace lcpb200
