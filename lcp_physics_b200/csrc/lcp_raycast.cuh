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
// kept in registers. The scene's bodies are staged through shared memory in tiles (TC circles; up to TP polygons of at
// most TV vertices, with their orientation and edge normals computed once per tile), so any world size works. Every
// thread visits the bodies in index order and only a strictly nearer hit replaces the best: the result depends neither
// on the chunking nor on the tile sizes. No atomics.
#pragma once
#include "lcp_ray_launch.h"

namespace lcpb200 {
namespace ray {

constexpr int NT = 256;       // rays per CTA at most (blockDim.x = R rounded up to a warp, capped at NT)
constexpr int TC = 256;       // circles per tile
constexpr int TV = 1024;      // polygon vertices per tile (>= 4 polygons at nv = 256)
constexpr int TP = 256;       // polygons per tile

// Tile staging shared by raycast_kernel and sdf_kernel (lcp_sdf.cuh). Every thread of the CTA calls these with the same
// arguments, between a barrier that frees the shared memory and one that publishes the tile.
//
// nb, nv are bd.nb, bd.nv and tid, nth threadIdx.x, blockDim.x, passed in from the kernel's registers.
//
// Circles c0 .. c0 + n - 1 of scene sc: centre, radius and active flag (aw: the scene's active words, or nullptr).
template <typename T>
__device__ __forceinline__ void stage_circles(const cts::Bodies<T>& bd, int nb, int sc, int c0, int n,
                                              const uint32_t* aw, T* s_cx, T* s_cy, T* s_cr, unsigned char* s_con,
                                              int tid, int nth) {
  for (int k = tid; k < n; k += nth) {
    const size_t g = (size_t)sc * nb + c0 + k;
    const int b = c0 + k;
    s_cx[k] = bd.pos[2 * g]; s_cy[k] = bd.pos[2 * g + 1]; s_cr[k] = bd.rad[g];
    s_con[k] = aw ? (unsigned char)((__ldg(aw + (b >> 5)) >> (b & 31)) & 1u) : (unsigned char)1;
  }
}

// Polygons q0 .. q0 + n - 1 of scene sc (bodies nb + q0 + k, dynamic polygons then obstacles): the vertices (polygon q
// at s_pv[2 q nv]), the orientation s_po[q] (+-1 from poly_orient; 0: inactive), and per edge e the flag s_eok[q nv + e]
// (edge_ok) and the outward unit normal s_pn[2 (q nv + e)] (zero for a zero-length edge). Holds two barriers of its own.
template <typename T>
__device__ __forceinline__ void stage_polygons(const cts::Bodies<T>& bd, int nb, int nv, int sc, int q0, int n,
                                               const uint32_t* aw, T* s_pv, T* s_pn, unsigned char* s_eok,
                                               signed char* s_po, int tid, int nth) {
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
}

// the polygons of one tile: as many as fit TV vertices, at most TP
__host__ __device__ __forceinline__ int poly_tile(int npo, int nv) { return npo > 0 ? (TV / nv < TP ? TV / nv : TP) : 1; }

template <typename T>
__global__ void __launch_bounds__(NT) raycast_kernel(RayArgs<T> a, int chunks) {
  __shared__ T s_cx[TC], s_cy[TC], s_cr[TC];
  __shared__ unsigned char s_con[TC];           // circle active
  __shared__ T s_pv[2 * TV];                    // vertices of the tile's polygons, polygon q at 2 q nv
  __shared__ T s_pn[2 * TV];                    // outward unit normal of edge e of polygon q, at 2 (q nv + e)
  __shared__ unsigned char s_eok[TV];           // edge of non-zero length
  __shared__ signed char s_po[TP];              // orientation (+-1), 0: inactive polygon
  const int tid = threadIdx.x, nth = blockDim.x;
  const cts::Bodies<T>& bd = a.bd;
  const int nb = bd.nb, npo = bd.np + bd.no, nv = bd.nv;
  const int nt = nb + npo, words = (nt + 31) >> 5;
  const int ptile = poly_tile(npo, nv);
  const T maxd = a.max_dist;
  const long long items = (long long)a.B * chunks;
  for (long long it = blockIdx.x; it < items; it += gridDim.x) {
    const int sc = (int)(it / chunks);
    const int r = (int)(it - (long long)sc * chunks) * nth + tid;
    const bool live = r < a.R;
    const size_t ri = (size_t)sc * a.R + (live ? r : 0);
    T ux = T(0), oy = T(0), ox = T(0), uy = T(0);       // this order keeps the SASS of before the staging helpers
    if (live) {
      ox = a.origin[2 * ri]; oy = a.origin[2 * ri + 1];
      ux = a.dir[2 * ri]; uy = a.dir[2 * ri + 1];
    }
    const bool valid = live && isfinite(ox) && isfinite(oy) && isfinite(ux) && isfinite(uy) && ux * ux + uy * uy > T(0);
    const uint32_t* aw = a.active ? a.active + (size_t)sc * words : nullptr;
    T best = maxd, bnx = T(0), bny = T(0);
    int bbody = -1, bfeat = -1;
    // ---- circles
    for (int c0 = 0; c0 < nb; c0 += TC) {
      const int n = nb - c0 < TC ? nb - c0 : TC;
      __syncthreads();                                   // the previous tile (or work item) is done with the smem
      stage_circles(bd, nb, sc, c0, n, aw, s_cx, s_cy, s_cr, s_con, tid, nth);
      __syncthreads();
      if (valid) {
        for (int k = 0; k < n; ++k) {
          if (!s_con[k]) continue;
          const T wx = ox - s_cx[k], wy = oy - s_cy[k], rr = s_cr[k];
          const T b = ux * wx + uy * wy;
          const T kk = wx * wx + wy * wy - rr * rr;
          if (kk < T(0) || b >= T(0)) continue;
          const T disc = b * b - kk;
          if (disc < T(0)) continue;
          const T t = kk / (-b + sqrt(disc));
          if (bbody < 0 ? t <= best : t < best) {
            best = t; bbody = c0 + k; bfeat = -1;
            bnx = (wx + t * ux) / rr; bny = (wy + t * uy) / rr;
          }
        }
      }
    }
    // ---- polygons, then obstacles (polygon q is body nb + q)
    for (int q0 = 0; q0 < npo; q0 += ptile) {
      const int n = npo - q0 < ptile ? npo - q0 : ptile;
      __syncthreads();
      stage_polygons(bd, nb, nv, sc, q0, n, aw, s_pv, s_pn, s_eok, s_po, tid, nth);
      __syncthreads();
      if (valid) {
        for (int q = 0; q < n; ++q) {
          if (!s_po[q]) continue;
          const T* P = &s_pv[2 * q * nv];
          const T* N = &s_pn[2 * q * nv];
          const unsigned char* ok = &s_eok[q * nv];
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
          if (miss || fe < 0 || !(te >= T(0) && te <= tl)) continue;
          if (bbody < 0 ? te <= best : te < best) {
            best = te; bbody = nb + q0 + q; bfeat = fe;
            bnx = N[2 * fe]; bny = N[2 * fe + 1];
          }
        }
      }
    }
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
