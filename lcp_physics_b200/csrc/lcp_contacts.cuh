// lcp_contacts.cuh -- batched contact detection for scenes of circles (SURVEY.md section 8 row f-2).
//
// Restates the circle-circle branch of the reference's contact handler (physics/contacts.py:68-80) together
// with the pair enumeration of World.find_contacts (physics/world.py:139-142: the broadphase callback visits
// every pair of geoms once):
//     r = rad_i + rad_j;  dist = |pos_i - pos_j|;  penetration = r - dist;  contact iff penetration >= -eps.
// One CTA per scene walks all nb (nb - 1) / 2 pairs (i < j) in lexicographic order -- the order in which the
// reference appends to world.contacts for circle scenes, which fixes the row order of Jc / Jf / E and therefore
// the LCP the engine builds -- and compacts the touching pairs IN THAT ORDER with a block-wide exclusive scan
// (ballot prefix inside a warp, warp totals through shared memory): deterministic, no atomics, no sort.
// Outputs: the pair list body1 / body2 [B, cap] (padded with the pair (0, 1)), and the TRUE number of touching
// pairs per scene (which may exceed cap: the caller checks). The contact geometry (normal, p1, p2, penetration)
// is evaluated by the caller on the selected pairs only (O(cap), differentiable in torch), so this kernel
// replaces the O(nb^2) part: at nb = 513 it tests 131 328 pairs per scene.
// The same kernels take static convex polygon obstacles (lcpb200_world_contacts): the walk then also visits the
// circle-obstacle pairs (i, nb + k), in the order of a reference World whose bodies are [circles..., obstacles...],
// with the circle-hull rule of contacts.py:84-144; no == 0 is the circle-only walk.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace lcpb200 {
namespace cts {

constexpr int NT = 256;
constexpr int ITEMS = 4;            // consecutive pairs per thread and chunk

// number of pairs (i', j') with i' < i, i.e. index of pair (i, i + 1), in a list of nt bodies
__device__ __forceinline__ long long pairs_before(long long i, long long nt) { return i * (2 * nt - i - 1) / 2; }

// Circle (centre cx, cy) against the static convex polygon P[nv][2] (world frame, either orientation), restating the
// circle-hull branch of the reference's contact handler (contacts.py:84-144). The reference finds the closest point
// with a GJK seeded by random.choice; the closest point of a convex polygon is unique, so it is computed here edge by
// edge (first edge wins a tie). Zero-length edges (a vertex repeated to pad a polygon to the batch's V) are skipped.
//   inside == false: the centre is outside; (qx, qy) is the closest point and d2 its squared distance.
//   inside == true:  SAT branch: the edge of largest separation sep = n . (c - v_e) (outward unit normal n, first
//                    edge wins a tie; the reference starts its scan at the edge that won last time), normal (nx, ny).
template <typename T>
struct PolyHit {
  bool inside;
  T d2, qx, qy;       // outside
  T sep, nx, ny;      // inside
};

template <typename T>
__device__ __forceinline__ PolyHit<T> circle_polygon(const T* __restrict__ P, int nv, T cx, T cy) {
  T area = T(0);
  for (int e = 0; e < nv; ++e) {
    const int f = e + 1 == nv ? 0 : e + 1;
    area += P[2 * e] * P[2 * f + 1] - P[2 * e + 1] * P[2 * f];
  }
  const T orient = area > T(0) ? T(1) : T(-1);       // outward normal = orient * (ey, -ex) / |e|
  PolyHit<T> h;
  h.d2 = T(INFINITY); h.qx = cx; h.qy = cy;
  h.sep = T(-INFINITY); h.nx = T(0); h.ny = T(0);
  bool inside = true;
  for (int e = 0; e < nv; ++e) {
    const int f = e + 1 == nv ? 0 : e + 1;
    const T ax = P[2 * e], ay = P[2 * e + 1];
    const T ex = P[2 * f] - ax, ey = P[2 * f + 1] - ay;
    const T len = sqrt(ex * ex + ey * ey);
    if (!(len > T(0))) continue;                     // a repeated vertex (padding to the common V): no edge
    const T nx = orient * ey / len, ny = -orient * ex / len;
    const T sp = nx * (cx - ax) + ny * (cy - ay);
    if (sp > T(0)) inside = false;
    if (sp > h.sep) { h.sep = sp; h.nx = nx; h.ny = ny; }
    T t = ((cx - ax) * ex + (cy - ay) * ey) / (ex * ex + ey * ey);
    t = t < T(0) ? T(0) : (t > T(1) ? T(1) : t);
    const T qx = ax + t * ex, qy = ay + t * ey;
    const T d2 = (cx - qx) * (cx - qx) + (cy - qy) * (cy - qy);
    if (d2 < h.d2) { h.d2 = d2; h.qx = qx; h.qy = qy; }
  }
  h.inside = inside;
  return h;
}

// One CTA per scene walks the pairs of the body list [circles 0..nb-1, obstacles nb..nb+no-1] in lexicographic
// order: pair (i, j), i < nb, i < j < nb + no -- circle-circle pairs (j < nb) and circle-obstacle pairs (j >= nb);
// obstacles never pair with each other. no == 0 is the circle-only walk of lcpb200_find_contacts.
// verts: [B, no, nv, 2] world-frame polygon vertices (nullptr when no == 0).
template <typename T>
__global__ void __launch_bounds__(NT) find_contacts_kernel(int B, int nb, int no, int nv, int cap, T eps,
                                                           const T* __restrict__ pos, const T* __restrict__ rad,
                                                           const T* __restrict__ verts, int32_t* __restrict__ body1,
                                                           int32_t* __restrict__ body2, int32_t* __restrict__ counts) {
  __shared__ int warp_tot[NT / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nt = nb + no;                                        // bodies in the pair list
  const long long npairs = pairs_before(nb, nt);                 // rows i < nb; no == 0: nb (nb - 1) / 2
  const int imax = nb - 1 < nt - 2 ? nb - 1 : nt - 2;            // last row with a pair
  for (int sc = blockIdx.x; sc < B; sc += gridDim.x) {
    const T* P = pos + (size_t)sc * nb * 2;
    const T* R = rad + (size_t)sc * nb;
    const T* V = no > 0 ? verts + (size_t)sc * no * nv * 2 : nullptr;
    int32_t* o1 = body1 + (size_t)sc * cap;
    int32_t* o2 = body2 + (size_t)sc * cap;
    int base = 0;                                                // touching pairs found in the previous chunks
    for (long long q0 = 0; q0 < npairs; q0 += (long long)NT * ITEMS) {
      const long long q = q0 + (long long)tid * ITEMS;
      int i = 0, j = 0;
      if (q < npairs) {                                          // (i, j) of pair q: closed form + exact fix-up
        const double t = 2.0 * nt - 1.0;
        long long ii = (long long)floor((t - sqrt(t * t - 8.0 * (double)q)) * 0.5);
        if (ii < 0) ii = 0;
        if (ii > imax) ii = imax;
        while (ii + 1 <= imax && pairs_before(ii + 1, nt) <= q) ++ii;
        while (ii > 0 && pairs_before(ii, nt) > q) --ii;
        i = (int)ii;
        j = (int)(q - pairs_before(ii, nt)) + i + 1;
      }
      unsigned hit = 0;
      int pi[ITEMS], pj[ITEMS];
#pragma unroll
      for (int u = 0; u < ITEMS; ++u) {
        pi[u] = i; pj[u] = j;
        if (q + u < npairs) {
          if (j < nb) {
            const T dx = P[2 * i] - P[2 * j], dy = P[2 * i + 1] - P[2 * j + 1];
            const T dist = sqrt(dx * dx + dy * dy);
            const T pen = R[i] + R[j] - dist;                    // contacts.py:70-73
            if (!(pen < -eps)) hit |= 1u << u;                   // `if penetration < -eps: return`
          } else {
            const PolyHit<T> h = circle_polygon<T>(V + (size_t)(j - nb) * nv * 2, nv, P[2 * i], P[2 * i + 1]);
            // outside: `if best_dist > eps: return` (contacts.py:110-112); inside: sep - rad < 0 <= eps always
            if (h.inside || !(sqrt(h.d2) - R[i] > eps)) hit |= 1u << u;
          }
          if (++j == nt) { ++i; j = i + 1; }
        }
      }
      const int mine = __popc(hit);
      int incl = mine;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
      if (lane == 31) warp_tot[warp] = incl;
      __syncthreads();
      int before = base, total = 0;
#pragma unroll
      for (int w = 0; w < NT / 32; ++w) { const int v = warp_tot[w]; if (w < warp) before += v; total += v; }
      int at = before + incl - mine;
#pragma unroll
      for (int u = 0; u < ITEMS; ++u)
        if (hit & (1u << u)) { if (at < cap) { o1[at] = pi[u]; o2[at] = pj[u]; } ++at; }
      base += total;
      __syncthreads();                                           // warp_tot is rewritten by the next chunk
    }
    const int pad2 = nt > 1 ? 1 : 0;                             // padding: a valid pair, (0, 1)
    for (int k = base + tid; k < cap; k += NT) { o1[k] = 0; o2[k] = pad2; }
    if (tid == 0) counts[sc] = base;
  }
}

// Geometry of the selected pairs, for callers that do not need autograd through the contact generation.
// Circle-circle (contacts.py:69-77): normal = (pos1 - pos2) / dist, penetration = r1 + r2 - dist,
// p1 = -normal (r1 - pen / 2), p2 = normal (r2 - pen / 2).
// Circle-obstacle (body2 = nb + k, contacts.py:84-144; see circle_polygon): outside, with q the closest point,
// normal = (c - q) / |c - q|, p1 = q - c, p2 = q - oref_k, penetration = r - |c - q|; centre inside, with the
// separating edge (n, sep), normal = n, p1 = -n sep, q = c + p1, p2 = q - oref_k, penetration = r - sep.
// mu / restitution = mean of the two bodies' (world.py:144-151, :213-224). Unused slots (k >= counts[scene]) get the
// geometry of the padding pair and penetration = -1e30. oref [B, no, 2]: the obstacles' reference points;
// ofric / orest [B, no]: their friction and restitution.
template <typename T>
__global__ void __launch_bounds__(NT) contact_geometry_kernel(int B, int nb, int no, int nv, int cap,
                                                              const T* __restrict__ pos, const T* __restrict__ rad,
                                                              const T* __restrict__ fric, const T* __restrict__ rest,
                                                              const T* __restrict__ verts, const T* __restrict__ oref,
                                                              const T* __restrict__ ofric, const T* __restrict__ orest,
                                                              const int32_t* __restrict__ body1,
                                                              const int32_t* __restrict__ body2,
                                                              const int32_t* __restrict__ counts, T* __restrict__ normal,
                                                              T* __restrict__ p1, T* __restrict__ p2, T* __restrict__ pen,
                                                              T* __restrict__ mu, T* __restrict__ rest_c) {
  const long long total = (long long)B * cap;
  for (long long t = blockIdx.x * (long long)NT + threadIdx.x; t < total; t += (long long)gridDim.x * NT) {
    const int sc = (int)(t / cap), k = (int)(t - (long long)sc * cap);
    const int i = body1[t], j = body2[t];
    const T* P = pos + (size_t)sc * nb * 2;
    const T* R = rad + (size_t)sc * nb;
    if (j < nb) {
      const T dx = P[2 * i] - P[2 * j], dy = P[2 * i + 1] - P[2 * j + 1];
      const T dist = sqrt(dx * dx + dy * dy);
      const T r1 = R[i], r2 = R[j];
      const T pn = r1 + r2 - dist;
      const T nx = dx / dist, ny = dy / dist;
      const T a1 = r1 - pn / 2, a2 = r2 - pn / 2;
      normal[2 * t] = nx; normal[2 * t + 1] = ny;
      p1[2 * t] = -nx * a1; p1[2 * t + 1] = -ny * a1;
      p2[2 * t] = nx * a2; p2[2 * t + 1] = ny * a2;
      pen[t] = k < counts[sc] ? pn : T(-1e30);
      mu[t] = T(0.5) * (fric[(size_t)sc * nb + i] + fric[(size_t)sc * nb + j]);
      rest_c[t] = T(0.5) * (rest[(size_t)sc * nb + i] + rest[(size_t)sc * nb + j]);
    } else {
      const size_t ob = (size_t)sc * no + (j - nb);
      const T cx = P[2 * i], cy = P[2 * i + 1], r = R[i];
      const PolyHit<T> h = circle_polygon<T>(verts + ob * nv * 2, nv, cx, cy);
      T nx, ny, qx, qy, pn;
      if (h.inside) {
        nx = h.nx; ny = h.ny; pn = r - h.sep;
        qx = cx - nx * h.sep; qy = cy - ny * h.sep;             // best_pt2 = center + normal * -(dist + rad)
      } else {
        const T dist = sqrt(h.d2);
        qx = h.qx; qy = h.qy; pn = r - dist;
        nx = (cx - qx) / dist; ny = (cy - qy) / dist;
      }
      normal[2 * t] = nx; normal[2 * t + 1] = ny;
      p1[2 * t] = qx - cx; p1[2 * t + 1] = qy - cy;
      p2[2 * t] = qx - oref[2 * ob]; p2[2 * t + 1] = qy - oref[2 * ob + 1];
      pen[t] = k < counts[sc] ? pn : T(-1e30);
      mu[t] = T(0.5) * (fric[(size_t)sc * nb + i] + ofric[ob]);
      rest_c[t] = T(0.5) * (rest[(size_t)sc * nb + i] + orest[ob]);
    }
  }
}

template <typename T>
static void launch_contact_geometry(int B, int nb, int no, int nv, int cap, const T* pos, const T* rad, const T* fric,
                                    const T* rest, const T* verts, const T* oref, const T* ofric, const T* orest,
                                    const int32_t* body1, const int32_t* body2, const int32_t* counts, T* normal, T* p1,
                                    T* p2, T* pen, T* mu, T* rest_c, int num_sms, cudaStream_t st) {
  const long long total = (long long)B * cap;
  long long grid = (total + NT - 1) / NT;
  if (grid > 8LL * num_sms) grid = 8LL * num_sms;
  contact_geometry_kernel<T><<<(int)grid, NT, 0, st>>>(B, nb, no, nv, cap, pos, rad, fric, rest, verts, oref, ofric,
                                                        orest, body1, body2, counts, normal, p1, p2, pen, mu, rest_c);
}

template <typename T>
static void launch_find_contacts(int B, int nb, int no, int nv, int cap, T eps, const T* pos, const T* rad,
                                 const T* verts, int32_t* body1, int32_t* body2, int32_t* counts, int num_sms,
                                 cudaStream_t st) {
  const int grid = B < 8 * num_sms ? B : 8 * num_sms;
  find_contacts_kernel<T><<<grid, NT, 0, st>>>(B, nb, no, nv, cap, eps, pos, rad, verts, body1, body2, counts);
}

}  // namespace cts
}  // namespace lcpb200
