// lcp_contacts.cuh -- batched contact detection for scenes of circles and convex polygons (SURVEY.md section 8 row f-2).
//
// Restates the circle-circle branch of the reference's contact handler (physics/contacts.py:68-80) together
// with the pair enumeration of World.find_contacts (physics/world.py:139-142: the broadphase callback visits
// every pair of geoms once):
//     r = rad_i + rad_j;  dist = |pos_i - pos_j|;  penetration = r - dist;  contact iff penetration >= -eps.
// One CTA per scene walks all nb (nb - 1) / 2 pairs (i < j) in lexicographic order -- the order in which the
// reference appends to world.contacts for circle scenes, which fixes the row order of Jc / Jf / E and therefore
// the LCP the engine builds -- and compacts the contacts IN THAT ORDER with a block-wide exclusive scan of the
// per-thread contact counts (warp prefix through shuffles, warp totals through shared memory): deterministic, no
// atomics, no sort.
// Outputs: the pair list body1 / body2 [B, cap] (padded with the pair (0, 1), or (0, 0) when the list holds one
// body), and the TRUE number of contacts per
// scene (which may exceed cap: the caller checks). The contact geometry (normal, p1, p2, penetration) is evaluated
// on the selected pairs only (contact_geometry_kernel, or differentiable torch ops), so the walk replaces the
// O(nb^2) part: at nb = 513 it tests 131 328 pairs per scene.
// The body list is [circles 0..nb-1, dynamic polygons nb..nb+np-1, static obstacles nb+np..nb+np+no-1], the order of
// a reference World built from [Circle..., Rect / Hull..., pinned Rect / Hull...]:
//   * circle-polygon pairs (dynamic or static polygon) use the circle-hull rule of contacts.py:84-144;
//   * polygon-polygon and polygon-obstacle pairs use the hull-hull rule of contacts.py:145-292 (SAT both ways,
//     reference-face clipping): 0, 1 or 2 contacts per pair, stored in the order of the clipped points;
//   * obstacles never pair with each other.
// The walk is templated on HULLS: HULLS == false is the walk of lcpb200_contacts without feat (circles and
// obstacles, np == 0), one contact per pair at most. MASK == true (lcpb200_contacts with no_contact) reads a
// pair-exclusion bitmask shared by the batch and skips an excluded pair before
// any rule is evaluated, as the reference's `if geom1 in geom2.no_contact: return` (contacts.py:60, add_no_contact).
// ACTIVE == true (lcpb200_contacts_active) walks each scene over its own active bodies: the CTA first compacts the
// scene's active body indices into shared memory, then walks the pairs of that sub-list, so a scene pays for its own
// pairs only and its contacts come in the order of the world that holds just its active bodies.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace lcpb200 {
namespace cts {

constexpr int NT = 256;
constexpr int ITEMS = 4;            // consecutive pairs per thread and chunk
constexpr int MAX_NV = 256;         // vertices per polygon (feat packs edge indices in 8 bits)
constexpr int MAX_ACTIVE_NT = 8192; // bodies of a world walked with per-scene activity (uint16 list, 16 KB of smem)

// number of pairs (i', j') with i' < i, i.e. index of pair (i, i + 1), in a list of nt bodies
__host__ __device__ __forceinline__ long long pairs_before(long long i, long long nt) { return i * (2 * nt - i - 1) / 2; }

// The three body groups of one batch. Circles: pos [B,nb,2], rad / fric / rest [B,nb]. Dynamic polygons: world-frame
// vertices pverts [B,np,nv,2] (positive area), centroids pcen [B,np,2], pfric / prest [B,np]. Obstacles: world-frame
// vertices overts [B,no,nv,2] (either orientation), reference points (centroids) oref [B,no,2], ofric / orest [B,no].
// fric / rest / pfric / prest / ofric / orest are read by the geometry only.
template <typename T>
struct Bodies {
  int nb, np, no, nv;
  const T *pos, *rad, *fric, *rest;
  const T *pverts, *pcen, *pfric, *prest;
  const T *overts, *oref, *ofric, *orest;
  // polygon body b (nb <= b < nb + np + no) of scene sc: vertices and centroid / reference point
  __host__ __device__ __forceinline__ const T* verts(int sc, int b) const {
    return b < nb + np ? pverts + ((size_t)sc * np + (b - nb)) * nv * 2 : overts + ((size_t)sc * no + (b - nb - np)) * nv * 2;
  }
  __host__ __device__ __forceinline__ const T* centre(int sc, int b) const {
    return b < nb + np ? pcen + ((size_t)sc * np + (b - nb)) * 2 : oref + ((size_t)sc * no + (b - nb - np)) * 2;
  }
  __host__ __device__ __forceinline__ T friction(int sc, int b) const {
    return b < nb ? fric[(size_t)sc * nb + b] : b < nb + np ? pfric[(size_t)sc * np + b - nb] : ofric[(size_t)sc * no + b - nb - np];
  }
  __host__ __device__ __forceinline__ T restitution(int sc, int b) const {
    return b < nb ? rest[(size_t)sc * nb + b] : b < nb + np ? prest[(size_t)sc * np + b - nb] : orest[(size_t)sc * no + b - nb - np];
  }
};

// +1 for a polygon of positive shoelace area (its outward edge normals are left_orthogonal(e) = (ey, -ex), the
// orientation Hull asserts, bodies.py:169, :228-235), -1 otherwise
template <typename T>
__host__ __device__ __forceinline__ T poly_orient(const T* __restrict__ P, int nv) {
  T area = T(0);
  for (int e = 0; e < nv; ++e) {
    const int f = e + 1 == nv ? 0 : e + 1;
    area += P[2 * e] * P[2 * f + 1] - P[2 * e + 1] * P[2 * f];
  }
  return area > T(0) ? T(1) : T(-1);
}

// Circle (centre cx, cy) against the convex polygon P[nv][2] (world frame, either orientation), restating the
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
__host__ __device__ __forceinline__ PolyHit<T> circle_polygon(const T* __restrict__ P, int nv, T cx, T cy) {
  const T orient = poly_orient(P, nv);               // outward normal = orient * (ey, -ex) / |e|
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

// ------------------------------------------------------------------ hull-hull (contacts.py:145-292)
// feat of a hull-hull contact: the discrete choices of the rule, so that every geometry path (contact_geometry_kernel,
// the torch mirror in world.py) rebuilds the contact from the same features:
//   bits 0-1  the point: 0 / 1 = endpoint 0 / 1 of the incident edge, 2 = cut by the first clip plane, 3 = cut by
//             the second clip plane
//   bits 2-3  the outcome of the first clip: 0 = [v0, v1], 1 = [v0, cut], 2 = [v1, cut]
//   bit  4    1 iff body2 holds the reference face
//   bits 5-12 reference edge, bits 13-20 incident edge (edge e runs from vertex e to vertex e + 1 mod nv)
// Every other contact has feat -1.
__host__ __device__ __forceinline__ int pack_feat(int kind, int clip1, int ref2, int re, int ie) {
  return kind | clip1 << 2 | ref2 << 4 | re << 5 | ie << 13;
}

// P: the vertices, vertex v at P[2 v] -- a pointer, or a view that computes them on every read (ray::MovedVerts)
template <class V>
__host__ __device__ __forceinline__ bool edge_ok(V P, int nv, int e) {
  const int f = e + 1 == nv ? 0 : e + 1;
  const auto ex = P[2 * f] - P[2 * e], ey = P[2 * f + 1] - P[2 * e + 1];
  return sqrt(ex * ex + ey * ey) > decltype(ex)(0);
}

template <typename T>
struct Sep {
  T dist;
  int edge, sup;
};

// test_separations(hull1, hull2) (contacts.py:219-250): over the edges of P1 (outward unit normal n), the support
// vertex of P2 in direction -n (get_support, :207-217: `>=`, the last maximal vertex wins) and its distance
// n . (v2_sup - v1_e) to the edge; returns the edge of largest distance (first edge wins a tie: the reference
// starts its scan at the edge that won last time). The pair is separated iff dist > eps (the early exit of :239-241
// returns at the first edge that raises the running maximum above eps, so it fires iff the maximum is > eps).
// P1 / P2: pointers or vertex views, as in edge_ok.
template <typename T, class V1, class V2>
__host__ __device__ Sep<T> separation(V1 P1, T o1, V2 P2, int nv) {
  Sep<T> s;
  s.dist = T(-INFINITY); s.edge = 0; s.sup = 0;
  for (int e = 0; e < nv; ++e) {
    const int f = e + 1 == nv ? 0 : e + 1;
    const T ex = P1[2 * f] - P1[2 * e], ey = P1[2 * f + 1] - P1[2 * e + 1];
    const T len = sqrt(ex * ex + ey * ey);
    if (!(len > T(0))) continue;
    const T nx = o1 * ey / len, ny = -o1 * ex / len;
    T best = T(-INFINITY);
    int sup = 0;
    for (int v = 0; v < nv; ++v) {
      const T d = -(nx * P2[2 * v] + ny * P2[2 * v + 1]);
      if (d >= best) { best = d; sup = v; }
    }
    const T dist = nx * (P2[2 * sup] - P1[2 * e]) + ny * (P2[2 * sup + 1] - P1[2 * e + 1]);
    if (dist > s.dist) { s.dist = dist; s.edge = e; s.sup = sup; }
  }
  return s;
}

// get_incident_edge (contacts.py:253-267): of the two edges at vertex s of P (the last non-degenerate edge before it
// and the first from it), the one whose outward unit normal has the smallest dot product with the reference normal
// (the edge before s wins a tie)
template <typename T>
__host__ __device__ int incident_edge(const T* __restrict__ P, T o, int nv, int s, T nx, T ny) {
  int ep = s, en = s;
  for (int k = 1; k <= nv; ++k) { const int e = (s - k + nv) % nv; if (edge_ok(P, nv, e)) { ep = e; break; } }
  for (int k = 0; k < nv; ++k) { const int e = (s + k) % nv; if (edge_ok(P, nv, e)) { en = e; break; } }
  T best = T(1e10);
  int be = ep;
  for (int u = 0; u < 2; ++u) {
    const int e = u == 0 ? ep : en;
    const int f = e + 1 == nv ? 0 : e + 1;
    const T ex = P[2 * f] - P[2 * e], ey = P[2 * f + 1] - P[2 * e + 1];
    const T len = sqrt(ex * ex + ey * ey);
    const T dot = nx * (o * ey / len) + ny * (-o * ex / len);
    if (dot < best) { best = dot; be = e; }
  }
  return be;
}

// The reference face of a hull-hull pair and the incident edge clipped to it (clip_segment_to_line twice,
// contacts.py:270-292), in the reference body's frame (about its centroid cr, as the reference holds Hull.verts).
// Both clip planes pass at +-|e_ref| / 2 from the reference body's CENTROID along left_orthogonal(n), not about the
// edge's midpoint: for a non-symmetric hull the window is off-centre, as in the reference.
template <typename T>
struct Face {
  T nx, ny;               // outward unit normal of the reference edge
  T rx, ry;               // its first vertex
  T x[4], y[4];           // v0, v1 (incident edge), cut by the first plane, cut by the second plane
  int clip1;              // 0: [v0, v1], 1: [v0, cut], 2: [v1, cut], 3: fewer than two points (no contact)
  int second[2];          // the points kept by the second clip, in order (-1: none); at least one is kept
};

// clip1 < 0: the first clip's outcome from the signs, as the reference; otherwise the recorded outcome (feat)
template <typename T>
__host__ __device__ Face<T> clip_face(const T* __restrict__ Pr, T crx, T cry, T orr, int re, const T* __restrict__ Pi,
                                      int ie, int nv, int clip1) {
  Face<T> F;
  const int rf = re + 1 == nv ? 0 : re + 1;
  const T ex = Pr[2 * rf] - Pr[2 * re], ey = Pr[2 * rf + 1] - Pr[2 * re + 1];
  const T len = sqrt(ex * ex + ey * ey);
  F.nx = orr * ey / len; F.ny = -orr * ex / len;
  F.rx = Pr[2 * re] - crx; F.ry = Pr[2 * re + 1] - cry;
  const T h = len / 2;
  const int jf = ie + 1 == nv ? 0 : ie + 1;
  F.x[0] = Pi[2 * ie] - crx; F.y[0] = Pi[2 * ie + 1] - cry;
  F.x[1] = Pi[2 * jf] - crx; F.y[1] = Pi[2 * jf + 1] - cry;
  const T px = F.ny, py = -F.nx;                        // clip plane left_orthogonal(n)
  const T d0 = px * F.x[0] + py * F.y[0] + h, d1 = px * F.x[1] + py * F.y[1] + h;
  if (clip1 < 0) clip1 = d0 >= T(0) ? (d1 >= T(0) ? 0 : 1) : (d1 >= T(0) ? 2 : 3);
  F.clip1 = clip1;
  const T t1 = d0 / (d0 - d1);
  F.x[2] = F.x[0] + t1 * (F.x[1] - F.x[0]); F.y[2] = F.y[0] + t1 * (F.y[1] - F.y[0]);
  const int a = clip1 == 2 ? 1 : 0, b = clip1 == 0 ? 1 : 2;
  const T e0 = -px * F.x[a] + -py * F.y[a] + h, e1 = -px * F.x[b] + -py * F.y[b] + h;
  const T t2 = e0 / (e0 - e1);
  F.x[3] = F.x[a] + t2 * (F.x[b] - F.x[a]); F.y[3] = F.y[a] + t2 * (F.y[b] - F.y[a]);
  // second clip: [a if e0 >= 0] + [b if e1 >= 0] + [cut if the endpoints straddle the plane or < 2 points kept]
  F.second[0] = F.second[1] = -1;
  int k = 0;
  if (e0 >= T(0)) F.second[k++] = a;
  if (e1 >= T(0)) F.second[k++] = b;
  if (e0 * e1 < T(0) || k < 2) F.second[k < 2 ? k : 1] = 3;
  return F;
}

// distance of clipped point `kind` to the reference edge and its projection onto the edge's line (contacts.py:173-178)
template <typename T>
__host__ __device__ __forceinline__ T face_point(const Face<T>& F, int kind, T& qx, T& qy) {
  const T dist = F.nx * (F.x[kind] - F.rx) + F.ny * (F.y[kind] - F.ry);
  qx = F.x[kind] + F.nx * -dist; qy = F.y[kind] + F.ny * -dist;
  return dist;
}

// The hull-hull contacts of bodies P1 (body1, centroid c1) and P2 (body2): count 0..2 and their feat codes.
template <typename T>
__host__ __device__ int hull_hull(const T* __restrict__ P1, const T* __restrict__ c1, const T* __restrict__ P2,
                         const T* __restrict__ c2, int nv, T eps, int* feat) {
  const T o1 = poly_orient(P1, nv), o2 = poly_orient(P2, nv);
  const Sep<T> s1 = separation(P1, o1, P2, nv);
  if (!(s1.dist <= eps)) return 0;                                  // contacts.py:148-151
  const Sep<T> s2 = separation(P2, o2, P1, nv);
  if (!(s2.dist <= eps)) return 0;                                  // :152-155
  const int ref2 = s2.dist > s1.dist ? 1 : 0;                       // :156
  const T* Pr = ref2 ? P2 : P1;
  const T* Pi = ref2 ? P1 : P2;
  const T* cr = ref2 ? c2 : c1;
  const T orr = ref2 ? o2 : o1, oi = ref2 ? o1 : o2;
  const Sep<T>& s = ref2 ? s2 : s1;
  const int rf = s.edge + 1 == nv ? 0 : s.edge + 1;
  const T ex = Pr[2 * rf] - Pr[2 * s.edge], ey = Pr[2 * rf + 1] - Pr[2 * s.edge + 1];
  const T len = sqrt(ex * ex + ey * ey);
  const int ie = incident_edge(Pi, oi, nv, s.sup, orr * ey / len, -orr * ex / len);
  const Face<T> F = clip_face(Pr, cr[0], cr[1], orr, s.edge, Pi, ie, nv, -1);
  if (F.clip1 == 3) return 0;                                       // `if len(clipped_verts) < 2: return`
  int n = 0;
  for (int u = 0; u < 2; ++u) {
    const int kind = F.second[u];
    if (kind < 0) continue;
    T qx, qy;
    if (face_point(F, kind, qx, qy) <= eps) feat[n++] = pack_feat(kind, F.clip1, ref2, s.edge, ie);
  }
  return n;
}

// One CTA per scene walks the pairs (i, j), i < j, i < nb + np (a dynamic body), j < nb + np + no, in lexicographic
// order; obstacles never pair with each other. Each pair yields 0, 1 or 2 contacts (HULLS == false: 0 or 1).
// feat [B, cap] (HULLS only, may be nullptr): the hull-hull features, -1 for every other contact.
// no_contact (MASK only): bit i * nt + j (i < j, nt = nb + np + no) set iff the pair (i, j) never makes contact; an
// excluded pair sets no hit bit, so the compaction keeps the order of the remaining pairs.
// ACTIVE (with HULLS and MASK; nt <= MAX_ACTIVE_NT): active [B, ceil(nt / 32)] (nullptr: every body active), bit k of
// scene s set iff body k takes part in scene s. The scene's active bodies are listed in index order (dynamic bodies
// first, then obstacles, as in the body list); the pairs are enumerated over that list's counts (nd_s, nt_s) and
// mapped back to body indices, which everything after the decode uses (the mask, the rule dispatch, the outputs).
// no_contact may be nullptr; otherwise scene s reads its mask at no_contact + s * nc_stride (stride 0: one mask for
// the batch).
template <typename T, bool HULLS, bool MASK = false, bool ACTIVE = false>
__global__ void __launch_bounds__(NT) find_contacts_kernel(Bodies<T> bd, int B, int cap, T eps,
                                                           int32_t* __restrict__ body1, int32_t* __restrict__ body2,
                                                           int32_t* __restrict__ feat, int32_t* __restrict__ counts,
                                                           const uint32_t* __restrict__ no_contact = nullptr,
                                                           const uint32_t* __restrict__ active = nullptr,
                                                           long long nc_stride = 0) {
  static_assert(!ACTIVE || (HULLS && MASK), "the active walk is the polygon walk with a per-scene mask");
  __shared__ int warp_tot[NT / 32];
  __shared__ uint16_t act[ACTIVE ? MAX_ACTIVE_NT : 1];           // ACTIVE: the scene's active bodies, in index order
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nb = bd.nb, nv = bd.nv;
  const int nd = nb + (HULLS ? bd.np : 0);                       // dynamic bodies: the rows of the pair list
  const int nt = nd + bd.no;                                     // bodies in the pair list
  long long npairs = pairs_before(nd, nt);                       // rows i < nd; circles only: nb (nb - 1) / 2
  int imax = nd - 1 < nt - 2 ? nd - 1 : nt - 2;                  // last row with a pair
  int ntw = nt;                                                  // length of the list the pairs are decoded over
  for (int sc = blockIdx.x; sc < B; sc += gridDim.x) {
    const T* P = bd.pos + (size_t)sc * nb * 2;
    const T* R = bd.rad + (size_t)sc * nb;
    int32_t* o1 = body1 + (size_t)sc * cap;
    int32_t* o2 = body2 + (size_t)sc * cap;
    const uint32_t* mask = no_contact;
    if constexpr (ACTIVE) {
      // compaction of the scene's active bodies: one 32-body word per thread (nt <= 8192 = 32 NT), a block-wide
      // exclusive scan of (active bodies | active dynamic bodies << 16) per word
      if (mask) mask += (size_t)sc * nc_stride;
      const int words = (nt + 31) >> 5;
      uint32_t w = 0;
      if (tid < words) {
        w = active ? __ldg(active + (size_t)sc * words + tid) : 0xffffffffu;
        const int left = nt - 32 * tid;                          // bodies in this word
        if (left < 32) w &= (1u << left) - 1u;
      }
      const int dleft = nd - 32 * tid;                           // dynamic bodies in this word
      const uint32_t wd = dleft >= 32 ? w : dleft <= 0 ? 0u : w & ((1u << dleft) - 1u);
      const int mine = __popc(w) | __popc(wd) << 16;
      int incl = mine;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
      __syncthreads();                                           // the previous scene is done with act and warp_tot
      if (lane == 31) warp_tot[warp] = incl;
      __syncthreads();
      int before = 0, total = 0;
#pragma unroll
      for (int w8 = 0; w8 < NT / 32; ++w8) { const int v = warp_tot[w8]; if (w8 < warp) before += v; total += v; }
      int at = (before + incl - mine) & 0xffff;
      for (uint32_t r = w; r; r &= r - 1u) act[at++] = (uint16_t)(32 * tid + __ffs(r) - 1);
      __syncthreads();                                           // act complete; warp_tot is rewritten by the walk
      const int nd_s = total >> 16;
      ntw = total & 0xffff;
      npairs = pairs_before(nd_s, ntw);
      imax = nd_s - 1 < ntw - 2 ? nd_s - 1 : ntw - 2;
    }
    int base = 0;                                                // contacts found in the previous chunks
    for (long long q0 = 0; q0 < npairs; q0 += (long long)NT * ITEMS) {
      const long long q = q0 + (long long)tid * ITEMS;
      int i = 0, j = 0;
      if (q < npairs) {                                          // (i, j) of pair q: closed form + exact fix-up
        const double t = 2.0 * ntw - 1.0;
        long long ii = (long long)floor((t - sqrt(t * t - 8.0 * (double)q)) * 0.5);
        if (ii < 0) ii = 0;
        if (ii > imax) ii = imax;
        while (ii + 1 <= imax && pairs_before(ii + 1, ntw) <= q) ++ii;
        while (ii > 0 && pairs_before(ii, ntw) > q) --ii;
        i = (int)ii;
        j = (int)(q - pairs_before(ii, ntw)) + i + 1;
      }
      unsigned hit = 0;                                          // HULLS: 2 bits per pair, its contact count
      int pi[ITEMS], pj[ITEMS];
      int f[HULLS ? 2 * ITEMS : 1];
#pragma unroll
      for (int u = 0; u < ITEMS; ++u) {
        int bi = i, bj = j;                                      // body indices of list positions (i, j)
        if constexpr (ACTIVE) {
          if (q + u < npairs) { bi = act[i]; bj = act[j]; }
        }
        pi[u] = bi; pj[u] = bj;
        if (q + u < npairs) {
          bool skip = false;
          if constexpr (MASK) {
            const long long bit = (long long)bi * nt + bj;
            if (!ACTIVE || mask) skip = (__ldg(mask + (bit >> 5)) >> (bit & 31)) & 1u;
          }
          if (skip) {
            if constexpr (HULLS) f[2 * u] = -1;
          } else if (bj < nb) {
            const T dx = P[2 * bi] - P[2 * bj], dy = P[2 * bi + 1] - P[2 * bj + 1];
            const T dist = sqrt(dx * dx + dy * dy);
            const T pen = R[bi] + R[bj] - dist;                  // contacts.py:70-73
            if (!(pen < -eps)) hit |= 1u << (HULLS ? 2 * u : u); // `if penetration < -eps: return`
            if constexpr (HULLS) f[2 * u] = -1;
          } else if (!HULLS || bi < nb) {
            const T* V = HULLS ? bd.verts(sc, bj) : bd.overts + ((size_t)sc * bd.no + (bj - nb)) * nv * 2;
            const PolyHit<T> h = circle_polygon<T>(V, nv, P[2 * bi], P[2 * bi + 1]);
            // outside: `if best_dist > eps: return` (contacts.py:110-112); inside: sep - rad < 0 <= eps always
            if (h.inside || !(sqrt(h.d2) - R[bi] > eps)) hit |= 1u << (HULLS ? 2 * u : u);
            if constexpr (HULLS) f[2 * u] = -1;
          } else if constexpr (HULLS) {
            const int n = hull_hull<T>(bd.verts(sc, bi), bd.centre(sc, bi), bd.verts(sc, bj), bd.centre(sc, bj), nv,
                                       eps, &f[2 * u]);
            hit |= (unsigned)n << (2 * u);
          }
          if (++j == ntw) { ++i; j = i + 1; }
        }
      }
      int mine;
      if constexpr (HULLS) {
        mine = 0;
#pragma unroll
        for (int u = 0; u < ITEMS; ++u) mine += (hit >> (2 * u)) & 3u;
      } else {
        mine = __popc(hit);
      }
      int incl = mine;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
      if (lane == 31) warp_tot[warp] = incl;
      __syncthreads();
      int before = base, total = 0;
#pragma unroll
      for (int w = 0; w < NT / 32; ++w) { const int v = warp_tot[w]; if (w < warp) before += v; total += v; }
      int at = before + incl - mine;
      if constexpr (HULLS) {
        int32_t* of = feat ? feat + (size_t)sc * cap : nullptr;
#pragma unroll
        for (int u = 0; u < ITEMS; ++u) {
          const int n = (hit >> (2 * u)) & 3;
          for (int c = 0; c < n; ++c) {
            if (at < cap) { o1[at] = pi[u]; o2[at] = pj[u]; if (of) of[at] = f[2 * u + c]; }
            ++at;
          }
        }
      } else {
#pragma unroll
        for (int u = 0; u < ITEMS; ++u)
          if (hit & (1u << u)) { if (at < cap) { o1[at] = pi[u]; o2[at] = pj[u]; } ++at; }
      }
      base += total;
      __syncthreads();                                           // warp_tot is rewritten by the next chunk
    }
    const int pad2 = nt > 1 ? 1 : 0;                             // padding: (0, 1), or (0, 0) for one body
    for (int k = base + tid; k < cap; k += NT) {
      o1[k] = 0; o2[k] = pad2;
      if (HULLS && feat) feat[(size_t)sc * cap + k] = nb == 0 ? 0 : -1;   // a hull-hull padding pair: edge 0, v0
    }
    if (tid == 0) counts[sc] = base;
  }
}

// Geometry of the selected pairs, for callers that do not need autograd through the contact generation.
// Circle-circle (contacts.py:69-77): normal = (pos1 - pos2) / dist, penetration = r1 + r2 - dist,
// p1 = -normal (r1 - pen / 2), p2 = normal (r2 - pen / 2).
// Circle-polygon (body2 = a polygon or obstacle with centroid cen, contacts.py:84-144; see circle_polygon): outside,
// with q the closest point, normal = (c - q) / |c - q|, p1 = q - c, p2 = q - cen, penetration = r - |c - q|; centre
// inside, with the separating edge (n, sep), normal = n, p1 = -n sep, q = c + p1, p2 = q - cen, penetration = r - sep.
// Hull-hull (feat >= 0, contacts.py:156-201): the clipped point v of feat in the reference body's frame, dist =
// n . (v - v_ref), pt = v - n dist; reference = body2: normal = n, p1 = pt + c2 - c1, p2 = pt; reference = body1:
// normal = -n, p1 = pt, p2 = pt + c1 - c2; penetration = -dist.
// mu / restitution = mean of the two bodies' (world.py:144-151, :213-224). Unused slots (k >= counts[scene]) get the
// geometry of the padding pair and penetration = -1e30; the pair (0, 0) of one circle gets the normal (1, 0) (a unit
// offset instead of 0 / 0), so every slot is finite.
template <typename T, bool HULLS>
__global__ void __launch_bounds__(NT) contact_geometry_kernel(Bodies<T> bd, int B, int cap,
                                                              const int32_t* __restrict__ body1,
                                                              const int32_t* __restrict__ body2,
                                                              const int32_t* __restrict__ feat,
                                                              const int32_t* __restrict__ counts, T* __restrict__ normal,
                                                              T* __restrict__ p1, T* __restrict__ p2, T* __restrict__ pen,
                                                              T* __restrict__ mu, T* __restrict__ rest_c) {
  const int nb = bd.nb, nv = bd.nv;
  const long long total = (long long)B * cap;
  for (long long t = blockIdx.x * (long long)NT + threadIdx.x; t < total; t += (long long)gridDim.x * NT) {
    const int sc = (int)(t / cap), k = (int)(t - (long long)sc * cap);
    const int i = body1[t], j = body2[t];
    const T* P = bd.pos + (size_t)sc * nb * 2;
    const T* R = bd.rad + (size_t)sc * nb;
    T nx, ny, a1x, a1y, a2x, a2y, pn;
    if (j < nb) {
      // the padding pair (0, 0) of a one-body list gets a unit offset, as _geometry_torch: finite, never a contact
      const T dx = i != j ? P[2 * i] - P[2 * j] : T(1), dy = i != j ? P[2 * i + 1] - P[2 * j + 1] : T(0);
      const T dist = sqrt(dx * dx + dy * dy);
      const T r1 = R[i], r2 = R[j];
      pn = r1 + r2 - dist;
      nx = dx / dist; ny = dy / dist;
      const T a1 = r1 - pn / 2, a2 = r2 - pn / 2;
      a1x = -nx * a1; a1y = -ny * a1;
      a2x = nx * a2; a2y = ny * a2;
    } else if (i < nb) {
      const T* cen = bd.centre(sc, j);
      const T cx = P[2 * i], cy = P[2 * i + 1], r = R[i];
      const PolyHit<T> h = circle_polygon<T>(bd.verts(sc, j), nv, cx, cy);
      T qx, qy;
      if (h.inside) {
        nx = h.nx; ny = h.ny; pn = r - h.sep;
        qx = cx - nx * h.sep; qy = cy - ny * h.sep;             // best_pt2 = center + normal * -(dist + rad)
      } else {
        const T dist = sqrt(h.d2);
        qx = h.qx; qy = h.qy; pn = r - dist;
        nx = (cx - qx) / dist; ny = (cy - qy) / dist;
      }
      a1x = qx - cx; a1y = qy - cy;
      a2x = qx - cen[0]; a2y = qy - cen[1];
    } else {
      if constexpr (!HULLS) continue;
      const int fc = feat[t] < 0 ? 0 : feat[t];
      const int kind = fc & 3, clip1 = (fc >> 2) & 3, ref2 = (fc >> 4) & 1, re = (fc >> 5) & 255, ie = (fc >> 13) & 255;
      const int br = ref2 ? j : i, bi = ref2 ? i : j;
      const T* Pr = bd.verts(sc, br);
      const T* cr = bd.centre(sc, br);
      const T* ci = bd.centre(sc, bi);
      const Face<T> F = clip_face(Pr, cr[0], cr[1], poly_orient(Pr, nv), re, bd.verts(sc, bi), ie, nv,
                                  clip1 > 2 ? 0 : clip1);
      T qx, qy;
      const T dist = face_point(F, kind, qx, qy);
      const T sx = qx + cr[0] - ci[0], sy = qy + cr[1] - ci[1];  // pt2 = pt1 + ref.pos - inc.pos
      pn = -dist;
      if (ref2) { nx = F.nx; ny = F.ny; a1x = sx; a1y = sy; a2x = qx; a2y = qy; }
      else { nx = -F.nx; ny = -F.ny; a1x = qx; a1y = qy; a2x = sx; a2y = sy; }
    }
    normal[2 * t] = nx; normal[2 * t + 1] = ny;
    p1[2 * t] = a1x; p1[2 * t + 1] = a1y;
    p2[2 * t] = a2x; p2[2 * t + 1] = a2y;
    pen[t] = k < counts[sc] ? pn : T(-1e30);
    mu[t] = T(0.5) * (bd.friction(sc, i) + bd.friction(sc, j));
    rest_c[t] = T(0.5) * (bd.restitution(sc, i) + bd.restitution(sc, j));
  }
}

template <typename T, bool HULLS>
static void launch_contact_geometry(const Bodies<T>& bd, int B, int cap, const int32_t* body1, const int32_t* body2,
                                    const int32_t* feat, const int32_t* counts, T* normal, T* p1, T* p2, T* pen, T* mu,
                                    T* rest_c, int num_sms, cudaStream_t st) {
  const long long total = (long long)B * cap;
  long long grid = (total + NT - 1) / NT;
  if (grid > 8LL * num_sms) grid = 8LL * num_sms;
  contact_geometry_kernel<T, HULLS><<<(int)grid, NT, 0, st>>>(bd, B, cap, body1, body2, feat, counts, normal, p1, p2,
                                                               pen, mu, rest_c);
}

template <typename T, bool HULLS, bool MASK = false>
static void launch_find_contacts(const Bodies<T>& bd, int B, int cap, T eps, int32_t* body1, int32_t* body2,
                                 int32_t* feat, int32_t* counts, int num_sms, cudaStream_t st,
                                 const uint32_t* no_contact = nullptr) {
  const int grid = B < 8 * num_sms ? B : 8 * num_sms;
  find_contacts_kernel<T, HULLS, MASK><<<grid, NT, 0, st>>>(bd, B, cap, eps, body1, body2, feat, counts, no_contact);
}

// the walk over each scene's active bodies (nt <= MAX_ACTIVE_NT); active / no_contact may be nullptr
template <typename T>
static void launch_find_contacts_active(const Bodies<T>& bd, int B, int cap, T eps, int32_t* body1, int32_t* body2,
                                        int32_t* feat, int32_t* counts, int num_sms, cudaStream_t st,
                                        const uint32_t* no_contact, long long nc_stride, const uint32_t* active) {
  const int grid = B < 8 * num_sms ? B : 8 * num_sms;
  find_contacts_kernel<T, true, true, true><<<grid, NT, 0, st>>>(bd, B, cap, eps, body1, body2, feat, counts,
                                                                 no_contact, active, nc_stride);
}

}  // namespace cts
}  // namespace lcpb200
