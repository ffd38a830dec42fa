// lcp_raycast.cuh -- batched ray casts against the bodies of BatchedWorld scenes (lcpb200_raycast).
//
// A ray is an origin o and a unit direction u. It is cast against the body list [circles, dynamic polygons, obstacles]
// of its scene and hits a body only where it ENTERS it at some 0 <= t <= max_dist:
//   circle (c, r):    w = o - c, b = u . w, k = |w|^2 - r^2; a miss if k < 0 (origin inside), b >= 0 or
//                     disc = b^2 - k < 0, else t = k / (-b + sqrt(disc)) (the cancellation-free form of -b - sqrt(disc));
//                     feat -1, normal (w + t u) / r.
//   convex polygon:   Cyrus-Beck clipping against every edge of non-zero length (either orientation, poly_orient;
//                     zero-length padding edges skipped as edge_ok does). Edge e: outward unit normal n_e, start vertex
//                     v_e, num = n_e . (v_e - o), den = n_e . u. den == 0: a miss if num < 0, else the edge is ignored;
//                     den < 0: an entering edge, t = num / den, the largest wins (the first on a tie); den > 0: a leaving
//                     edge, the smallest t is kept. A hit iff an entering edge exists and 0 <= t_enter <= t_leave,
//                     t_enter <= max_dist; feat = the entering edge, normal = its n_e. An origin inside has t_enter < 0.
// The nearest hit wins, an exact tie goes to the lower body index. No hit: body -1, feat -1, t = max_dist, normal 0.
// A direction of zero length or with a non-finite component, or a non-finite origin, hits nothing. Inactive bodies
// (active bit clear) are invisible.
//
// Layout: one CTA per (scene, chunk of blockDim.x rays) work item, one ray per thread, the best (t, body, feat, normal)
// kept in registers. The scene's bodies are staged through shared memory in tiles by SceneWalk, so any world size
// works. Every thread visits the bodies in index order and only a strictly nearer hit replaces the best: the result
// depends neither on the chunking nor on the tile sizes. No atomics.
#pragma once
#include "lcp_ray_launch.h"

namespace lcpb200 {
namespace ray {

constexpr int NT = 256;       // rays per CTA at most (blockDim.x = R rounded up to a warp, capped at NT)
constexpr int TC = 256;       // circles per tile
constexpr int TV = 1024;      // polygon vertices per tile (>= 4 polygons at nv = 256)
constexpr int TP = 256;       // polygons per tile

// The scene walk of raycast_kernel, sdf_kernel (lcp_sdf.cuh) and distance_kernel's nearest mode (lcp_distance.cuh).
// A kernel builds it once, before its grid-stride loop, so that the walk's constants are computed once per thread.
// Every thread of the CTA then calls it with the same scene sc and active words aw (nullptr: every body active). It
// stages the scene's bodies through shared memory in tiles: TC circles (centre, radius, active flag), then as many
// polygons (dynamic polygons, then obstacles; polygon q is body nb + q) as fit TV vertices, at most TP, with their
// orientation and edge normals computed once per tile. Between the barriers, a thread with `visit` set is called back
// in body index order, inactive bodies skipped:
//   circle(b, cx, cy, r)       circle b;
//   polygon(b, P, N, ok, o)    polygon b: vertex e at P[2 e], its edge's outward unit normal at N[2 e] (zero for a
//                              zero-length edge) and flag ok[e] (edge_ok), orientation o (+-1, poly_orient).
// Each tile is a __shared__ array of its own, so that ptxas drops the ones a kernel never reads.
template <typename T>
struct SceneWalk {
  const cts::Bodies<T>& bd;
  int tid, nth;
  int nb, npo, nv;
  int nt, words;                                // bodies, and 32-bit words of a scene's active mask
  int ptile;                                    // polygons per tile

  __device__ __forceinline__ explicit SceneWalk(const cts::Bodies<T>& b)
      : bd(b), tid(threadIdx.x), nth(blockDim.x), nb(b.nb), npo(b.np + b.no), nv(b.nv), nt(nb + npo),
        words((nt + 31) >> 5), ptile(npo > 0 ? (TV / nv < TP ? TV / nv : TP) : 1) {}

  template <class OnCircle, class OnPolygon>
  __device__ __forceinline__ void operator()(int sc, const uint32_t* aw, bool visit, OnCircle&& circle,
                                             OnPolygon&& polygon) const {
    __shared__ T s_cx[TC], s_cy[TC], s_cr[TC];
    __shared__ unsigned char s_con[TC];         // circle active
    __shared__ T s_pv[2 * TV];                  // vertices of the tile's polygons, polygon q at 2 q nv
    __shared__ T s_pn[2 * TV];                  // outward unit normal of edge e of polygon q, at 2 (q nv + e)
    __shared__ unsigned char s_eok[TV];         // edge of non-zero length
    __shared__ signed char s_po[TP];            // orientation (+-1), 0: inactive polygon
    // ---- circles
    for (int c0 = 0; c0 < nb; c0 += TC) {
      const int n = nb - c0 < TC ? nb - c0 : TC;
      __syncthreads();                                   // the previous tile (or work item) is done with the smem
      for (int k = tid; k < n; k += nth) {
        const size_t g = (size_t)sc * nb + c0 + k;
        const int b = c0 + k;
        s_cx[k] = bd.pos[2 * g]; s_cy[k] = bd.pos[2 * g + 1]; s_cr[k] = bd.rad[g];
        s_con[k] = aw ? (unsigned char)((__ldg(aw + (b >> 5)) >> (b & 31)) & 1u) : (unsigned char)1;
      }
      __syncthreads();
      if (visit) {
        for (int k = 0; k < n; ++k)
          if (s_con[k]) circle(c0 + k, s_cx[k], s_cy[k], s_cr[k]);
      }
    }
    // ---- polygons, then obstacles
    for (int q0 = 0; q0 < npo; q0 += ptile) {
      const int n = npo - q0 < ptile ? npo - q0 : ptile;
      __syncthreads();
      for (int k = tid; k < n * nv; k += nth) {
        const int q = k / nv, v = k - q * nv;
        const T* P = bd.verts(sc, nb + q0 + q);
        s_pv[2 * k] = P[2 * v]; s_pv[2 * k + 1] = P[2 * v + 1];
      }
      __syncthreads();
      for (int q = tid; q < n; q += nth) {
        const int b = nb + q0 + q;
        const bool on = !aw || ((__ldg(aw + (b >> 5)) >> (b & 31)) & 1u);
        s_po[q] = on ? (signed char)cts::poly_orient(&s_pv[2 * q * nv], nv) : (signed char)0;
      }
      __syncthreads();
      for (int k = tid; k < n * nv; k += nth) {
        const int q = k / nv, e = k - q * nv, f = e + 1 == nv ? 0 : e + 1;
        const T* P = &s_pv[2 * q * nv];
        const bool ok = cts::edge_ok(P, nv, e);
        const T ex = P[2 * f] - P[2 * e], ey = P[2 * f + 1] - P[2 * e + 1];
        const T len = sqrt(ex * ex + ey * ey);
        const T o = T(s_po[q]);
        s_eok[k] = ok;
        s_pn[2 * k] = ok ? o * ey / len : T(0);
        s_pn[2 * k + 1] = ok ? -o * ex / len : T(0);
      }
      __syncthreads();
      if (visit) {
        for (int q = 0; q < n; ++q)
          if (s_po[q]) polygon(nb + q0 + q, &s_pv[2 * q * nv], &s_pn[2 * q * nv], &s_eok[q * nv], (int)s_po[q]);
      }
    }
  }
};

template <typename T>
__global__ void __launch_bounds__(NT) raycast_kernel(RayArgs<T> a, int chunks) {
  const SceneWalk<T> walk(a.bd);
  const int tid = walk.tid, nth = walk.nth, nv = walk.nv;
  const T maxd = a.max_dist;
  const long long items = (long long)a.B * chunks;
  for (long long it = blockIdx.x; it < items; it += gridDim.x) {
    const int sc = (int)(it / chunks);
    const int r = (int)(it - (long long)sc * chunks) * nth + tid;
    const bool live = r < a.R;
    const size_t ri = (size_t)sc * a.R + (live ? r : 0);
    T ox = T(0), oy = T(0), ux = T(0), uy = T(0);
    if (live) {
      ox = a.origin[2 * ri]; oy = a.origin[2 * ri + 1];
      ux = a.dir[2 * ri]; uy = a.dir[2 * ri + 1];
    }
    const bool valid = live && isfinite(ox) && isfinite(oy) && isfinite(ux) && isfinite(uy) && ux * ux + uy * uy > T(0);
    const uint32_t* aw = a.active ? a.active + (size_t)sc * walk.words : nullptr;
    T best = maxd, bnx = T(0), bny = T(0);
    int bbody = -1, bfeat = -1;
    walk(sc, aw, valid,
      [&](int j, T cx, T cy, T rr) {
        const T wx = ox - cx, wy = oy - cy;
        const T b = ux * wx + uy * wy;
        const T kk = wx * wx + wy * wy - rr * rr;
        if (kk < T(0) || b >= T(0)) return;
        const T disc = b * b - kk;
        if (disc < T(0)) return;
        const T t = kk / (-b + sqrt(disc));
        if (bbody < 0 ? t <= best : t < best) {
          best = t; bbody = j; bfeat = -1;
          bnx = (wx + t * ux) / rr; bny = (wy + t * uy) / rr;
        }
      },
      [&](int j, const T* P, const T* N, const unsigned char* ok, int) {
        T te = T(-INFINITY), tl = T(INFINITY);
        int fe = -1;
        bool miss = false;
        for (int e = 0; e < nv; ++e) {
          if (!ok[e]) continue;
          const T nx = N[2 * e], ny = N[2 * e + 1];
          const T num = nx * (P[2 * e] - ox) + ny * (P[2 * e + 1] - oy);
          const T den = nx * ux + ny * uy;
          if (den == T(0)) {
            if (num < T(0)) { miss = true; break; }
            continue;
          }
          const T t = num / den;
          if (den < T(0)) {
            if (t > te) { te = t; fe = e; }
          } else if (t < tl) {
            tl = t;
          }
        }
        if (miss || fe < 0 || !(te >= T(0) && te <= tl)) return;
        if (bbody < 0 ? te <= best : te < best) {
          best = te; bbody = j; bfeat = fe;
          bnx = N[2 * fe]; bny = N[2 * fe + 1];
        }
      });
    if (live) {
      a.t[ri] = best;
      a.body[ri] = bbody;
      a.feat[ri] = bfeat;
      if (a.normal) { a.normal[2 * ri] = bnx; a.normal[2 * ri + 1] = bny; }
    }
  }
}

}  // namespace ray
}  // namespace lcpb200
