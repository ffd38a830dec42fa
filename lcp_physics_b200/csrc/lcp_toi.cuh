// lcp_toi.cuh -- batched times of impact between moving, rotating bodies of BatchedWorld scenes
// (lcpb200_time_of_impact).
//
// Motion: over tau in [0, 1] dynamic body k moves as p_k + tau D_k, D = (dth, dx, dy) in the layout of p (the motion
// of a step, start_p + v dt). A circle's centre moves (its rotation is irrelevant: dth is read as 0); a polygon's
// vertices at tau are c + tau dc + R(tau dth)(v0 - c), v0 its vertices and c its centre at tau = 0; obstacles stay.
// d(tau) is the body distance of distance_kernel (lcp_distance.cuh) between the two bodies at their poses at tau.
//
// Conservative advancement from tau = 0: at each iterate d(tau), its unit normal n (world, from A towards B) and
//   mu = -n . (dc_B - dc_A) + |dth_A| R_A + |dth_B| R_B
// (R_k: the largest |v0 - c| of a polygon, 0 for a circle or an obstacle) bound how fast d can fall. Then:
//   d - gap <= tol:                      a hit at tau;
//   mu <= 0 or tau + (d - gap) / mu > 1: no hit;
//   otherwise                            tau += (d - gap) / mu.
// The step never passes the first tau at which d reaches gap, so the reported tau is never later than the contact.
// TOI_MAX_ITER evaluations at most: a pair that reaches the cap reports the tau it reached as a hit (dist shows that
// d - gap > tol). A pair with d(0) < skip is not seen, one with d(0) == skip only when mu > 0 (sweep's convention: new
// contacts, not existing ones). A pair whose bodies do not move, or with a non-finite motion row, is not seen.
//
// Frame: d is evaluated in A's frame at tau = 0. A stays; B is moved by the relative rigid motion
// T_A(0) T_A(tau)^-1 T_B(tau) T_B(0)^-1, a rotation by phi = tau (dth_B - dth_A) about c_B and a shift s, read
// through MovedVerts (lcp_sdf.cuh) so that pair_distance, point_polygon and cts::separation run unchanged. At tau = 0
// the view returns the stored vertices exactly, so d(0) is distance_kernel's value. n and point_a are mapped back by
// T_A(tau) T_A(0)^-1.
//
// Pair mode reads (body_a, body_b) per query; first mode reads body_a and walks every other active body of the scene
// not excluded by no_contact (SceneWalk, obstacles included), in index order: from best = 1, body -1, a body replaces
// the best iff (body < 0 ? tau <= best : tau < best); a candidate is dropped once its next iterate passes the best hit
// (it could not replace it). Outputs: frac = tau (1 on a miss), body (-1), feat (dist_feat of the pair at tau, -1),
// dist = d at tau, normal and point_a (world, at tau), zeros on a miss.
//
// Layout: that of distance_kernel, one CTA per (scene, chunk of blockDim.x queries) work item, one query per thread,
// the best hit in registers; each candidate's motion row and centre are read from global memory by index. No atomics;
// the result depends neither on the chunking nor on the tile sizes.
#pragma once
#include "lcp_distance.cuh"

namespace lcpb200 {
namespace ray {

constexpr int TOI_MAX_ITER = 64;    // distance evaluations per pair at most

// A body's motion over the step: centre c at tau = 0, (dth, dx, dy), reach R
template <typename T>
struct Motion {
  T cx, cy, th, x, y, reach;
};

// the motion of body b of scene sc: false for a non-finite motion row. P: a polygon's vertices at tau = 0 (for R).
template <typename T>
__device__ __forceinline__ bool load_motion(const ToiArgs<T>& a, int sc, int b, const T* P, Motion<T>& m) {
  const cts::Bodies<T>& bd = a.bd;
  const int nd = bd.nb + bd.np;
  m.cx = m.cy = m.th = m.x = m.y = m.reach = T(0);
  if (b < bd.nb) {
    const size_t g = (size_t)sc * bd.nb + b;
    m.cx = bd.pos[2 * g]; m.cy = bd.pos[2 * g + 1];
  } else if (b < nd) {
    const size_t g = (size_t)sc * bd.np + (b - bd.nb);
    m.cx = bd.pcen[2 * g]; m.cy = bd.pcen[2 * g + 1];
  }
  if (b < nd) {
    const T* D = a.motion + ((size_t)sc * nd + b) * 3;
    m.th = b < bd.nb ? T(0) : D[0];
    m.x = D[1]; m.y = D[2];
    if (!(isfinite(D[0]) && isfinite(m.x) && isfinite(m.y))) return false;
    if (b >= bd.nb) {
      T r2 = T(0);
      for (int v = 0; v < bd.nv; ++v) {
        const T wx = P[2 * v] - m.cx, wy = P[2 * v + 1] - m.cy;
        r2 = fmax(r2, wx * wx + wy * wy);
      }
      m.reach = sqrt(r2);
    }
  }
  return true;
}

template <typename T>
__device__ __forceinline__ bool still(const Motion<T>& m) { return m.th == T(0) && m.x == T(0) && m.y == T(0); }

// A pair's time of impact and the distance choices at it
template <typename T>
struct Impact {
  T tau, d;
  T nx, ny, px, py;       // world normal (A towards B) and point_a at tau
  int feat;
};

// The advancement of A (static side at tau = 0, motion ma) against B (a circle (cx, cy, r), or polygon P of
// orientation o; motion mb) up to lim: true and the impact on a hit
template <typename T>
__device__ __forceinline__ bool advance(const Side<T, LoadedEdges<T>>& A, const Motion<T>& ma, bool bcircle, T r,
                                        const T* P, T o, const Motion<T>& mb, int nv, T gap, T skip, T tol, T lim,
                                        Impact<T>& out) {
  if (still(ma) && still(mb)) return false;
  const T abx = ma.cx - mb.cx, aby = ma.cy - mb.cy;      // c_A - c_B and c_B - c_A, exact negatives: s = 0 at tau = 0
  const T bax = mb.cx - ma.cx, bay = mb.cy - ma.cy;
  const T dcx = mb.x - ma.x, dcy = mb.y - ma.y, dth = mb.th - ma.th;
  const T rot = fabs(ma.th) * ma.reach + fabs(mb.th) * mb.reach;
  T tau = T(0);
  for (int it = 0; it < TOI_MAX_ITER; ++it) {
    const T ca = cos(tau * ma.th), sa = sin(tau * ma.th);
    const T qx = bax + tau * dcx, qy = bay + tau * dcy;   // c_B(tau) - c_A(tau)
    const T sx = abx + (ca * qx + sa * qy), sy = aby + (ca * qy - sa * qx);   // c_A + R(-alpha) q - c_B
    const T phi = tau * dth;
    const MovedVerts<T> mv{P, cos(phi) - T(1), sin(phi), mb.cx, mb.cy, sx, sy};
    const Side<T, LoadedEdges<T, MovedVerts<T>>> Bm{bcircle, mb.cx + sx, mb.cy + sy, r,
                                                    LoadedEdges<T, MovedVerts<T>>{mv, o, nv}, o};
    const Pair<T> p = pair_distance(A, Bm, nv);
    if (!isfinite(p.d)) return false;
    const T ux = p.mlen > T(0) ? p.mx / p.mlen : T(0), uy = p.mlen > T(0) ? p.my / p.mlen : T(0);
    const T sg = (p.feat >> 17) & 1 ? T(1) : T(-1);
    const T nx0 = sg * ux, ny0 = sg * uy;
    const T nx = ca * nx0 - sa * ny0, ny = sa * nx0 + ca * ny0;        // R(alpha) n0
    const T mu = -(nx * dcx + ny * dcy) + rot;
    if (it == 0 && (p.d < skip || (p.d == skip && !(mu > T(0))))) return false;
    const T gp = p.d - gap;
    if (gp <= tol || it + 1 == TOI_MAX_ITER) {
      const T wx = (p.x - p.w * ux) - ma.cx, wy = (p.y - p.w * uy) - ma.cy;   // point_a - c_A in A's frame
      out.tau = tau; out.d = p.d; out.nx = nx; out.ny = ny; out.feat = p.feat;
      out.px = ma.cx + tau * ma.x + (ca * wx - sa * wy);
      out.py = ma.cy + tau * ma.y + (sa * wx + ca * wy);
      return true;
    }
    if (!(mu > T(0))) return false;
    const T next = tau + gp / mu;
    if (!(next <= lim)) return false;
    tau = next;
  }
  return false;
}

template <typename T>
__global__ void __launch_bounds__(NT) toi_kernel(ToiArgs<T> a, int chunks) {
  const SceneWalk<T> walk(a.bd);
  const cts::Bodies<T>& bd = a.bd;
  const int tid = walk.tid, nth = walk.nth, nv = walk.nv, nt = walk.nt;
  const bool first = a.body_b == nullptr;
  const T gap = a.gap, skip = a.skip, tol = a.tol;
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
    const int ib = live && !first ? a.body_b[qi] : -1;
    bool valid = live && on(ia) && (first || (ib != ia && on(ib)));
    const Side<T, LoadedEdges<T>> A = load_body(bd, sc, valid ? ia : 0);
    Motion<T> ma;
    valid = load_motion(a, sc, valid ? ia : 0, A.g.P, ma) && valid;
    T best = T(1);
    int bbody = -1;
    Impact<T> bi;
    bi.d = bi.nx = bi.ny = bi.px = bi.py = T(0); bi.feat = -1;
    auto visit = [&](int j, bool circle, T r_, const T* P, T o) {
      Motion<T> mb;
      if (!load_motion(a, sc, j, P, mb)) return;
      Impact<T> im;
      if (!advance(A, ma, circle, r_, P, o, mb, nv, gap, skip, tol, bbody < 0 ? T(1) : best, im)) return;
      if (bbody < 0 ? im.tau <= best : im.tau < best) { best = im.tau; bbody = j; bi = im; }
    };
    if (!first) {
      if (valid) {
        const Side<T, LoadedEdges<T>> Bs = load_body(bd, sc, ib);
        visit(ib, Bs.circle, Bs.r, Bs.g.P, Bs.o);
      }
    } else {
      const uint32_t* nc = a.no_contact ? a.no_contact + (size_t)sc * a.nc_stride : nullptr;
      auto excluded = [&](int j) {
        if (!nc) return false;
        const long long bit = (long long)(ia < j ? ia : j) * nt + (ia < j ? j : ia);
        return ((__ldg(nc + (bit >> 5)) >> (bit & 31)) & 1u) != 0u;
      };
      walk(sc, aw, valid,
        [&](int j, T, T, T cr) {
          if (j == ia || excluded(j)) return;
          visit(j, true, cr, nullptr, T(0));
        },
        [&](int j, const T* P, const T*, const unsigned char*, int o) {
          if (j == ia || excluded(j)) return;
          visit(j, false, T(0), P, T(o));
        });
    }
    if (live) {
      const bool hit = bbody >= 0;
      a.frac[ri] = best;
      a.body[ri] = bbody;
      a.feat[ri] = hit ? bi.feat : -1;
      a.dist[ri] = hit ? bi.d : T(0);
      a.normal[2 * ri] = hit ? bi.nx : T(0);
      a.normal[2 * ri + 1] = hit ? bi.ny : T(0);
      a.point_a[2 * ri] = hit ? bi.px : T(0);
      a.point_a[2 * ri + 1] = hit ? bi.py : T(0);
    }
  }
}

}  // namespace ray
}  // namespace lcpb200
