// lcp_banded.cuh -- the engine's LCP for LARGE single scenes (SURVEY.md section 8 row f-3, BASELINE config 4:
// one World of hundreds of bodies, n = 3 nb in the thousands, m = 4 nc up to ~10^4), fp64.
//
// Same algorithm as lcp_condensed.cuh -- the reference's PDIPM (lcp/solvers/pdipm.py:49-179) with every
// Newton system solved through the condensed KKT matrix
//     [[K, A^T], [A, 0]],   K = Q + G^T (F + diag(s/z))^-1 G        (n + e unknowns instead of m)
// -- but K is no longer dense: block (i, j) of K is non-zero iff bodies i and j touch (world.py:172-211: a
// contact row of G has two bodies). The kernel orders the bodies by a breadth-first (Cuthill-McKee) sweep of
// the contact graph, which makes K BANDED (half bandwidth ~ 3 x the widest BFS level; a 2-D pile of 512 balls:
// ~100), moves the few bodies that break the band (pinned bodies: the floor touches a whole row of balls;
// anything with > DEGB contacts) together with the equality rows into a dense BORDER of <= 16 rows, and
// factors the resulting arrow matrix by a right-looking blocked LU without pivoting (K + border is
// quasi-definite, DESIGN.md section 3.1) that slides a (bw + 8 + 16)^2 window through shared memory:
// 8 pivots per pass, 2 N bw^2 flops instead of 2/3 N^3 (17 MFLOP instead of 2.4 GFLOP at N = 1539).
// The factors stream to an L2-resident workspace and come back, chunk by chunk and double buffered, for the
// substitutions (one warp solves while the others fetch). One CTA per scene, persistent grid; B large scenes
// run on B SMs.
//
// Everything per-row (z, s, residuals, W blocks) lives in an L2-resident per-CTA workspace: at m ~ 8000 the
// vectors alone (9 m doubles) exceed shared memory. Inputs are the engine's contact structure-of-arrays
// (lcpb200_engine_forward); nothing dense is ever formed.
#pragma once
#include "lcp_device.cuh"
#include "lcp_condensed.cuh"

namespace lcpb200 {
namespace bnd {

constexpr int NT = 256;
constexpr int BD = 16;            // border rows (3 per border body + equality rows), identity padded
constexpr int PV = 8;             // pivots per LU pass
constexpr int DEGB = 12;          // a body with more contacts than this is moved to the border
constexpr int EPT = 12;           // registers per thread for the rows / columns entering the window
constexpr int STATUS_UNSUPPORTED = -100;

struct BPlan {
  int ok;
  int nb, n, ncap, cs, m, e;      // m = cs * ncap: stride of lam / slack
  int nbp;                        // roundup(n, 8)
  int bwa_max;                    // largest supported active width (multiple of 8)
  int smem_bytes, win_bytes;
  int o_red, o_sv, o_rank, o_cf, o_sol, o_lp, o_up, o_win;         // shared memory (bytes)
  long long g_qd, g_ps, g_x, g_dx, g_rx, g_y, g_dy, g_ry, g_cg, g_z, g_s, g_d, g_rz, g_rs, g_dz, g_ds, g_t, g_h,
      g_W, g_E, g_Kb, g_KbT, g_Brow, g_Bcol, g_Cn, g_FB, g_doubles;  // per-CTA L2 workspace (doubles)
  long long i_deg, i_start, i_adj, i_ints;                            // per-CTA int workspace
};

inline long long bal2(long long x) { return (x + 1) & ~1LL; }

// Fills the offsets; returns false when the problem does not fit (shared memory).
inline bool carve_bplan(BPlan& P, int smem_limit) {
  const int n = P.n, nb = P.nb, ncap = P.ncap, cs = P.cs;
  P.nbp = (n + 7) & ~7;
  size_t o = 0;
  auto take = [&](int& f, size_t bytes) { f = (int)o; o += (bytes + 15) & ~(size_t)15; };
  take(P.o_red, 6 * 32 * 8);
  take(P.o_sv, 64 * 4);
  take(P.o_rank, (size_t)nb * 4);
  take(P.o_cf, BD * BD * 8);
  take(P.o_sol, (size_t)(P.nbp + BD) * 8);
  const long long fixed = (long long)o;
  // window (bwa + 8 + BD + 1)^2 doubles + two panels (bwa + BD) x 8; during the structure phase the window
  // region also holds the BFS arrays (3 nb + 1 + 2 ncap ints)
  int best = 0;
  for (int bwa = 8; bwa <= 128; bwa += 8) {                    // 128 = 32 SUBR rows per substitution round set
    const long long ldw = bwa + PV + BD + 1;
    const long long need = fixed + 2LL * (bwa + BD) * PV * 8 + 32 + ldw * ldw * 8;
    if (need > smem_limit) break;
    best = bwa;
  }
  if (best == 0) return false;
  P.bwa_max = best;
  take(P.o_lp, (size_t)(best + BD) * PV * 8);
  take(P.o_up, (size_t)(best + BD) * PV * 8);
  P.o_win = (int)o;
  P.win_bytes = (int)(((long long)smem_limit - (long long)o) & ~15LL);
  if ((long long)(3 * nb + 1 + 2 * ncap) * 4 + 8 + 28LL * nb > P.win_bytes) return false;   // + coordinates / candidate ranks
  P.smem_bytes = (int)o + P.win_bytes;
  long long g = 0;
  auto gt = [&](long long& f, long long cnt) { f = g; g += bal2(cnt); };
  gt(P.g_qd, n); gt(P.g_ps, n); gt(P.g_x, n); gt(P.g_dx, n); gt(P.g_rx, n);
  gt(P.g_y, BD); gt(P.g_dy, BD); gt(P.g_ry, BD);
  gt(P.g_cg, 12LL * ncap);
  const long long mr = (long long)cs * ncap;
  gt(P.g_z, mr); gt(P.g_s, mr); gt(P.g_d, mr); gt(P.g_rz, mr); gt(P.g_rs, mr); gt(P.g_dz, mr); gt(P.g_ds, mr);
  gt(P.g_t, mr); gt(P.g_h, mr);
  gt(P.g_W, 16LL * ncap); gt(P.g_E, 36LL * ncap);
  const long long ldk = best + 1;
  gt(P.g_Kb, (long long)P.nbp * ldk); gt(P.g_KbT, (long long)P.nbp * ldk);
  // border rows and columns interleaved: BB[i][0..15] = column i of the border rows, BB[i][16..31] = row i of the
  // border columns (one 256-byte line per entering index); g_Bcol is kept as the second half's offset
  gt(P.g_Brow, 2LL * BD * P.nbp); P.g_Bcol = P.g_Brow + (long long)BD * P.nbp; gt(P.g_Cn, BD * BD);
  const long long fbs = 72 + 2LL * PV * (best + BD);
  gt(P.g_FB, (long long)(P.nbp / PV) * fbs + BD * BD);
  P.g_doubles = g;
  long long gi = 0;
  auto it = [&](long long& f, long long cnt) { f = gi; gi += (cnt + 3) & ~3LL; };
  it(P.i_deg, nb); it(P.i_start, nb + 1); it(P.i_adj, 2LL * ncap);
  P.i_ints = gi;
  return true;
}

extern __shared__ __align__(16) unsigned char bnd_smem[];

struct BArgs {
  BPlan P;
  int B;
  cnd::EngineSoA<double> soa;
  const double *A, *b;
  double *zhat, *nu, *lam, *slack, *resid;
  int *status, *iters;
  double eps;
  int not_improved_lim, max_iter;
  double* wsd;                    // [grid][P.g_doubles]
  int* wsi;                       // [grid][P.i_ints]
  long long* prof;                // nullptr or [grid][BPH_COUNT]
};

// Backward (lcp/lcp.py:37-64) through the engine's assembly for large scenes: saved (zhat, nu, lam, slack) and
// dl/dzhat in, gradients w.r.t. the contact list out (same outputs as the condensed kernels' engine path).
struct BBwdArgs {
  BPlan P;
  int B;
  int R, chunks;                  // R cotangents, [R][B][...] slots, (scene, chunk) work items: as cnd::CBwdArgs
  cnd::EngineSoA<double> soa;
  const double* A;
  const double *zhat, *nu, *lam, *slack, *g;
  double *dmass, *dinertia, *dv, *dfext, *dnormal, *dp1, *dp2, *dmu, *drest, *dA, *db;   // any may be nullptr
  double* wsd;
  int* wsi;
  long long* prof;
  unsigned flags;                 // LCPB200_BWD_*: bit 0 = exact adjoint (transposed KKT system: K^T, W^T)
};

// Jacobian-vector products (lcpb200_engine_jvp_batched) for large scenes: saved solve and R tangents of the contact
// list in ([R][B][...], nullptr = zero), dz[R][B][n] out; (scene, chunk) work items as BBwdArgs.
struct BJvpArgs {
  BPlan P;
  int B;
  int R, chunks;
  cnd::EngineSoA<double> soa;
  const double* A;
  const double *zhat, *nu, *lam, *slack;
  cnd::EngineTangents<double> t;
  double* dz;
  double* wsd;
  int* wsi;
  long long* prof;
};

#ifdef LCP_BAND_DEVICE        // device code: compiled by lcp_band_kernels.cu only
enum { BPH_STRUCT = 0, BPH_WINV, BPH_ASSEMBLE, BPH_LU, BPH_RHS, BPH_SUBST, BPH_POST, BPH_RESID, BPH_STEP, BPH_GRADS,
       BPH_FACTORS, BPH_SOLVES, BPH_COUNT };   // same order as cnd::CPH_* (shared counter buffer)

struct BProf {
  long long* dst;
  long long t0;
  __device__ __forceinline__ void start(long long* d) { dst = d; if (dst) t0 = clock64(); }
  __device__ __forceinline__ void lap(int ph) {
    if (dst && threadIdx.x == 0) { const long long t = clock64(); atomicAdd((unsigned long long*)&dst[ph], (unsigned long long)(t - t0)); t0 = t; }
  }
  __device__ __forceinline__ void count(int ph, int k = 1) {
    if (dst && threadIdx.x == 0) atomicAdd((unsigned long long*)&dst[ph], (unsigned long long)k);
  }
};

// Per-scene context: pointers into shared memory / the L2 workspace and the sizes found at run time.
struct Ctx {
  double *win, *sol, *lp, *up, *red, *cf;
  int *rank, *sv;
  double *qd, *ps, *x, *dx, *rx, *y, *dy, *ry, *cg, *z, *s, *d, *rz, *rs, *dz, *ds, *t, *h, *W, *E, *Kb, *KbT, *Brow,
      *Bcol, *Cn, *FB;
  int *deg, *start, *adj;
  const int32_t *b1, *b2;
  const double* A;
  int nb, n, e, cs, ncap, nc, m;
  int nband, Nb, Nbp, nbb, nbd, bw, bwa, Wc, LDW, LP, fbs, npass, ldk, win_doubles, bwa_max;
  int o_win, o_sol, o_lp, o_up, o_cf;      // byte offsets of the shared-memory arrays (see smem_d)
};

// Pointer into the dynamic shared memory, derived from the __shared__ symbol INSIDE the function that uses it: a
// pointer that travels through Ctx (local memory) is generic, and the hot loops then compile to LD.E / ST.E with
// every store ordered against the next load (measured: the LU's trailing update ran at 10 DFMA per clock).
__device__ __forceinline__ double* smem_d(int byte_offset) { return reinterpret_cast<double*>(bnd_smem + byte_offset); }

// position of body `body`'s dof q in `sol` (band part first, then the border)
__device__ __forceinline__ int sol_index(const Ctx& c, int body, int q) {
  const int r = c.rank[body];
  return r >= 0 ? 3 * r + q : c.Nbp + 3 * (-1 - r) + q;
}

// ------------------------------------------------------------------ structure: geometry, adjacency, ordering
// Returns 0 = ok, 1 = unsupported topology, 2 = singular mass matrix.
__device__ __noinline__ int build_structure(Ctx& c, const cnd::EngineSoA<double>& E_, int sc) {
  const int tid = threadIdx.x, lane = tid & 31, nb = c.nb, n = c.n, e = c.e, ncs = E_.nc, cs = c.cs;
  const int nc = c.nc;
  const double* mass = E_.mass + (size_t)sc * nb;
  const double* inertia = E_.inertia + (size_t)sc * nb;
  const double* v = E_.v + (size_t)sc * n;
  const double* normal = E_.normal + (size_t)sc * ncs * 2;
  const double* p1 = E_.p1 + (size_t)sc * ncs * 2;
  const double* p2 = E_.p2 + (size_t)sc * ncs * 2;
  int* mark = reinterpret_cast<int*>(c.win);              // BFS arrays in the (idle) window region
  int* queue = mark + nb;
  int* startS = queue + nb;
  int* nbr = startS + nb + 1;
  // candidate orderings: coordinates of the bodies relative to the root of their component (integrated along the
  // BFS tree: pos_b2 - pos_b1 = p1 - p2 at a contact), component ids, ranks by x and by y
  double* px = reinterpret_cast<double*>(mark + ((3 * nb + 1 + 2 * c.ncap + 1) & ~1));
  double* py = px + nb;
  int* comp = reinterpret_cast<int*>(py + nb);
  int* rkx = comp + nb;
  int* rky = rkx + nb;
  int bad = 0;
  for (int j = tid; j < n; j += NT) {
    const int body = j / 3;
    const double q = (j - 3 * body == 0) ? inertia[body] : mass[body];      // world.py:57-61, bodies.py:44-47
    c.qd[j] = q;
    if (!(q != 0.0 && isfinite(q))) bad |= 2;
    c.ps[j] = E_.mode == 0 ? q * v[j] + E_.dt * E_.fext[(size_t)sc * n + j] : 0.0;   // engines.py:32 / :109
  }
  // queue[] (idle until the BFS) counts each body's one-body contacts: contacts with a static obstacle (body2 >= nb,
  // no dofs). They touch only body1's diagonal block, so they neither join the BFS graph nor send a body to the border.
  int* const nobst = queue;
  for (int bq = tid; bq < nb; bq += NT) { c.deg[bq] = 0; mark[bq] = 0; nobst[bq] = 0; }
  __syncthreads();
  for (int k = tid; k < nc; k += NT) {
    const int b1 = c.b1[k], b2 = c.b2[k];
    if (b1 == b2 || b1 < 0 || b2 < 0 || b1 >= nb) { bad |= 1; continue; }
    const bool two = b2 < nb;
    const double nx = normal[2 * k], ny = normal[2 * k + 1];
    const double p1x = p1[2 * k], p1y = p1[2 * k + 1], p2x = p2[2 * k], p2y = p2[2 * k + 1];
    double r1[3], r2[3];
    cnd::contact_row<double>(p1x, p1y, p2x, p2y, nx, ny, r1, r2);           // Jc row (world.py:172-184)
    if (!two) r2[0] = r2[1] = r2[2] = 0.0;
    const double v20 = two ? v[3 * b2] : 0.0, v21 = two ? v[3 * b2 + 1] : 0.0, v22 = two ? v[3 * b2 + 2] : 0.0;
    const double jv = r1[0] * v[3 * b1] + r1[1] * v[3 * b1 + 1] + r1[2] * v[3 * b1 + 2] +
                      r2[0] * v20 + r2[1] * v21 + r2[2] * v22;
    const double rc = E_.rest[(size_t)sc * ncs + k];
    double* g = c.cg + 12 * (size_t)k;
#pragma unroll
    for (int q = 0; q < 3; ++q) { g[q] = r1[q]; g[3 + q] = r2[q]; }
    if (E_.mode == 0) {
      c.h[k] = jv * rc;                                                     // engines.py:53,74
      cnd::contact_row<double>(p1x, p1y, p2x, p2y, ny, -nx, r1, r2);        // Jf rows: +- left_orthogonal(n)
      if (!two) r2[0] = r2[1] = r2[2] = 0.0;
#pragma unroll
      for (int q = 0; q < 3; ++q) { g[6 + q] = r1[q]; g[9 + q] = r2[q]; }
      c.h[c.ncap + k] = 0.0; c.h[2 * c.ncap + k] = 0.0; c.h[3 * c.ncap + k] = 0.0;
    } else {
      c.h[k] = jv + jv * -rc;                                               // engines.py:90
    }
    atomicAdd(&c.deg[b1], 1);
    if (two) atomicAdd(&c.deg[b2], 1);
    else atomicAdd(&nobst[b1], 1);
  }
  // bodies pinned by an equality row go to the border
  for (int t = tid; t < e * n; t += NT)
    if (c.A[t] != 0.0) mark[(t % n) / 3] = 1;
  const int anybad = __syncthreads_or(bad);
  if (anybad & 2) return 2;
  if (anybad & 1) return 1;
  // ---- CSR offsets (one warp: chunked inclusive scan) and the border list
  if (tid < 32) {
    int run = 0, nbb = 0;
    for (int b0 = 0; b0 < nb; b0 += 32) {
      const int bq = b0 + lane;
      const int dg = bq < nb ? c.deg[bq] : 0;
      int incl = dg;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(FULL, incl, o); if (lane >= o) incl += u; }
      if (bq < nb) { c.start[bq] = run + incl - dg; startS[bq] = run + incl - dg; }
      run += __shfl_sync(FULL, incl, 31);
      const bool isb = bq < nb && (mark[bq] != 0 || dg - nobst[bq] > DEGB);
      const unsigned bl = __ballot_sync(FULL, isb);
      if (isb) c.rank[bq] = -1 - (nbb + __popc(bl & ((1u << lane) - 1)));
      else if (bq < nb) c.rank[bq] = 0x7fffffff;                            // not placed yet
      nbb += __popc(bl);
    }
    if (lane == 0) { c.start[nb] = run; startS[nb] = run; c.sv[0] = nbb; }
  }
  __syncthreads();
  const int nbb = c.sv[0];
  if (3 * nbb + e > BD) return 1;
  for (int bq = tid; bq < nb; bq += NT) c.deg[bq] = 0;                      // reused as fill cursors
  __syncthreads();
  for (int k = tid; k < nc; k += NT) {
    const int b1 = c.b1[k], b2 = c.b2[k];
    c.adj[c.start[b1] + atomicAdd(&c.deg[b1], 1)] = 2 * k;
    if (b2 < nb) c.adj[c.start[b2] + atomicAdd(&c.deg[b2], 1)] = 2 * k + 1;
  }
  __syncthreads();
  // sort every list by contact index (deterministic gather order): short lists by one thread, long ones by rank
  for (int bq = tid; bq < nb; bq += NT) {
    const int s0 = startS[bq], dg = startS[bq + 1] - s0;
    if (dg > 32) continue;
    for (int i = 1; i < dg; ++i) {
      const int val = c.adj[s0 + i];
      int j = i - 1;
      while (j >= 0 && c.adj[s0 + j] > val) { c.adj[s0 + j + 1] = c.adj[s0 + j]; --j; }
      c.adj[s0 + j + 1] = val;
    }
  }
  __syncthreads();
  for (int bq = 0; bq < nb; ++bq) {
    const int s0 = startS[bq], dg = startS[bq + 1] - s0;
    if (dg <= 32) continue;                                                 // (uniform: everyone reads the same offsets)
    for (int i0 = 0; i0 < dg; i0 += NT) {                                   // rank sort through the nbr scratch
      const int i = i0 + tid;
      int val = 0, rk = 0;
      if (i < dg) {
        val = c.adj[s0 + i];
        for (int u = 0; u < dg; ++u) rk += (c.adj[s0 + u] < val);
        nbr[rk] = val;
      }
    }
    __syncthreads();
    for (int i = tid; i < dg; i += NT) c.adj[s0 + i] = nbr[i];
    __syncthreads();
  }
  // neighbour lists (body ids) for the BFS
  for (int bq = tid; bq < nb; bq += NT) {
    const int s0 = c.start[bq], s1 = c.start[bq + 1];
    for (int i = s0; i < s1; ++i) {
      const int a = c.adj[i], k = a >> 1, o = (a & 1) ? c.b1[k] : c.b2[k];
      nbr[i] = o < nb ? o : -1;                                             // -1: a static obstacle, not a graph node
    }
    mark[bq] = c.rank[bq] < 0 ? -2 : -1;                                    // -2 border, -1 unvisited, >= 0 position
  }
  __syncthreads();
  // ---- breadth-first ordering, level by level (warp 0). Two sweeps per component: the first finds a
  // far (pseudo-peripheral) body, the second, started there, is the ordering.
  if (tid < 32) {
    int tail = 0, ncomp = 0;
    for (int root = 0; root < nb; ++root) {
      if (mark[root] != -1) continue;
      int first = root;
      for (int sweep = 0; sweep < 2; ++sweep) {
        const int base = tail;
        __syncwarp();
        if (lane == 0) { queue[base] = first; mark[first] = base; px[first] = 0.0; py[first] = 0.0; comp[first] = ncomp; }
        __syncwarp();
        int hd = base, tl = base + 1, lvl_end = base + 1;
        while (hd < tl) {
          const int cnt = min(32, lvl_end - hd);
          const int u = lane < cnt ? queue[hd + lane] : -1;
          const int s0 = u >= 0 ? startS[u] : 0;
          const int dg = u >= 0 ? startS[u + 1] - s0 : 0;
          int maxd = dg;
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) maxd = max(maxd, __shfl_xor_sync(FULL, maxd, o));
          for (int k = 0; k < maxd; ++k) {
            const int w = k < dg ? nbr[s0 + k] : -1;
            const bool cand = w >= 0 && mark[w] == -1;
            const unsigned same = __match_any_sync(FULL, cand ? w : -1 - lane);
            const bool win = cand && (lane == __ffs(same) - 1);
            const unsigned wb = __ballot_sync(FULL, win);
            __syncwarp();                                                   // all reads of mark[] precede the winners' writes
            if (win) {
              const int pos = tl + __popc(wb & ((1u << lane) - 1));
              queue[pos] = w; mark[w] = pos; comp[w] = ncomp;
              const int ad = c.adj[s0 + k], kc = ad >> 1;
              const double ddx = p1[2 * kc] - p2[2 * kc], ddy = p1[2 * kc + 1] - p2[2 * kc + 1];
              px[w] = (ad & 1) ? px[u] - ddx : px[u] + ddx;
              py[w] = (ad & 1) ? py[u] - ddy : py[u] + ddy;
            }
            tl += __popc(wb);
            __syncwarp();
          }
          hd += cnt;
          if (hd == lvl_end) lvl_end = tl;
        }
        if (sweep == 0) {
          first = queue[tl - 1];
          __syncwarp();
          for (int i = base + lane; i < tl; i += 32) mark[queue[i]] = -1;   // undo, start again from the far body
          __syncwarp();
        } else {
          tail = tl;
        }
      }
      ++ncomp;
    }
    if (lane == 0) c.sv[1] = tail;
  }
  __syncthreads();
  const int nband = c.sv[1];
  // ---- two more candidate orderings: components one after the other, bodies of a component sorted by their x
  // (resp. y) coordinate (a pile that is long in one direction gets a band as wide as its SHORT side, where the
  // breadth-first fronts of a hexagonal packing are up to twice as wide). Rank sort, ties by body index.
  for (int bq = tid; bq < nb; bq += NT) {
    if (mark[bq] < 0) continue;
    const int cb = comp[bq];
    const double xb = px[bq], yb = py[bq];
    int rx_ = 0, ry_ = 0;
    for (int o = 0; o < nb; ++o) {
      if (mark[o] < 0) continue;
      const int co = comp[o];
      const double xo = px[o], yo = py[o];
      const bool cl = co < cb, ce = co == cb;
      rx_ += (cl || (ce && (xo < xb || (xo == xb && o < bq)))) ? 1 : 0;
      ry_ += (cl || (ce && (yo < yb || (yo == yb && o < bq)))) ? 1 : 0;
    }
    rkx[bq] = rx_; rky[bq] = ry_;
  }
  __syncthreads();
  int bw3[3] = {0, 0, 0};
  for (int k = tid; k < nc; k += NT) {
    const int u1 = c.b1[k], u2 = c.b2[k];
    if (u2 < nb && mark[u1] >= 0 && mark[u2] >= 0) {
      bw3[0] = max(bw3[0], abs(mark[u1] - mark[u2]));
      bw3[1] = max(bw3[1], abs(rkx[u1] - rkx[u2]));
      bw3[2] = max(bw3[2], abs(rky[u1] - rky[u2]));
    }
  }
  {
#pragma unroll
    for (int q = 0; q < 3; ++q)
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) bw3[q] = max(bw3[q], __shfl_xor_sync(FULL, bw3[q], o));
    int* ir = reinterpret_cast<int*>(c.red);
    if (lane == 0) { ir[3 * (tid >> 5)] = bw3[0]; ir[3 * (tid >> 5) + 1] = bw3[1]; ir[3 * (tid >> 5) + 2] = bw3[2]; }
    __syncthreads();
    bw3[0] = bw3[1] = bw3[2] = 0;
    for (int w = 0; w < NT / 32; ++w) { bw3[0] = max(bw3[0], ir[3 * w]); bw3[1] = max(bw3[1], ir[3 * w + 1]); bw3[2] = max(bw3[2], ir[3 * w + 2]); }
    __syncthreads();
  }
  const int* best = mark;
  int bwb = bw3[0];
  if (bw3[1] < bwb) { bwb = bw3[1]; best = rkx; }
  if (bw3[2] < bwb) { bwb = bw3[2]; best = rky; }
  for (int bq = tid; bq < nb; bq += NT) if (mark[bq] >= 0) c.rank[bq] = best[bq];
  __syncthreads();
  c.nband = nband; c.Nb = 3 * nband; c.Nbp = (c.Nb + 7) & ~7;
  c.nbb = nbb; c.nbd = 3 * nbb + e;
  c.bw = 3 * bwb + 2;
  c.bwa = (c.bw + 7) & ~7;
  c.Wc = c.bwa + PV;
  c.LDW = c.Wc + BD + 1;
  c.LP = c.bwa + BD;
  c.fbs = 72 + 2 * PV * c.LP;
  c.npass = c.Nbp / PV;
  c.ldk = c.bw + 1;
  // The plan sized the band rows (Kb / KbT: ldk <= bwa_max + 1), the panels, the factor blocks and the
  // substitution's rows (32 SUBR) for bwa <= bwa_max. The window check alone is not enough: the leftover shared
  // memory of a plan can hold the window of the next width up while the L2 workspace cannot hold its band.
  if (c.bwa > c.bwa_max) return 1;
  if ((long long)c.LDW * c.LDW > c.win_doubles) return 1;                    // band too wide for the window
  return 0;
}

// ------------------------------------------------------------------ W_c = (F_c + diag(1/d))^-1, E_c = Gd^T W Gd
// trans (exact-adjoint backward, mode 0): the transposed system, F_c^T in place of F_c. Its block is
// (F_c^T + diag(1/d))^-1 = W_c^T, so c.W receives W_c^T and E_c = Gd^T W_c^T Gd; the border ([A, 0] / [A^T; 0])
// is symmetric, so the band, the ordering and the LU are those of K^T unchanged. Mode 1 has F = 0 (W is a scalar):
// trans changes nothing there.
__device__ __forceinline__ void contact_blocks(const Ctx& c, int mode, const double* mu, bool trans) {
  const int ncap = c.ncap;
  for (int k = threadIdx.x; k < c.nc; k += NT) {
    const double* g = c.cg + 12 * (size_t)k;
    double gn[6], gf[6];
#pragma unroll
    for (int q = 0; q < 6; ++q) gn[q] = g[q];
    double* Eo = c.E + 36 * (size_t)k;
    if (mode != 0) {
      const double w = c.d[k];                                              // (0 + 1/d)^-1
      c.W[16 * (size_t)k] = w;
#pragma unroll
      for (int a = 0; a < 6; ++a)
#pragma unroll
        for (int b = 0; b < 6; ++b) Eo[a * 6 + b] = w * gn[a] * gn[b];
      continue;
    }
#pragma unroll
    for (int q = 0; q < 6; ++q) gf[q] = g[6 + q];
    // F = [[0,0,0,0],[0,0,0,1],[0,0,0,1],[mu,-1,-1,0]] on {normal, f1, f2, gamma}   (engines.py:66-73)
    double M[4][4] = {{0, 0, 0, 0}, {0, 0, 0, 1}, {0, 0, 0, 1}, {mu[k], -1, -1, 0}};
#pragma unroll
    for (int r = 0; r < 4; ++r) M[r][r] += 1.0 / c.d[r * ncap + k];
    unsigned swaps = 0;
    int bit = 0;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {                                        // Gauss-Jordan, partial pivoting, in registers
#pragma unroll
      for (int i = kk + 1; i < 4; ++i) {
        const bool sw = fabs(M[i][kk]) > fabs(M[kk][kk]);
        swaps |= (sw ? 1u : 0u) << bit;
        ++bit;
#pragma unroll
        for (int q = 0; q < 4; ++q) { const double u = M[kk][q], w = M[i][q]; M[kk][q] = sw ? w : u; M[i][q] = sw ? u : w; }
      }
      const double r = 1.0 / M[kk][kk];
      M[kk][kk] = 1.0;
#pragma unroll
      for (int q = 0; q < 4; ++q) M[kk][q] *= r;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (i == kk) continue;
        const double f = M[i][kk];
        M[i][kk] = 0.0;
#pragma unroll
        for (int q = 0; q < 4; ++q) M[i][q] = fma(-f, M[kk][q], M[i][q]);
      }
    }
#pragma unroll
    for (int kk = 3; kk >= 0; --kk) {
#pragma unroll
      for (int i = 3; i > kk; --i) {
        --bit;
        const bool sw = (swaps >> bit) & 1u;
#pragma unroll
        for (int q = 0; q < 4; ++q) { const double u = M[q][kk], w = M[q][i]; M[q][kk] = sw ? w : u; M[q][i] = sw ? u : w; }
      }
    }
    double* Wo = c.W + 16 * (size_t)k;
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int q = 0; q < 4; ++q) Wo[r * 4 + q] = trans ? M[q][r] : M[r][q];
    // rows of Gd: gn, gf, -gf, 0 (W^T swaps the two off-diagonal couplings)
    const double mnf = M[0][1] - M[0][2], mfn = M[1][0] - M[2][0];
    const double wnn = M[0][0], wnf = trans ? mfn : mnf, wfn = trans ? mnf : mfn;
    const double wff = M[1][1] - M[1][2] - M[2][1] + M[2][2];
#pragma unroll
    for (int a = 0; a < 6; ++a) {
      const double ra = wnn * gn[a] + wfn * gf[a], rb = wnf * gn[a] + wff * gf[a];
#pragma unroll
      for (int b = 0; b < 6; ++b) Eo[a * 6 + b] = ra * gn[b] + rb * gf[b];
    }
  }
}

// K(i, j) += val in the arrow storage. ri / rj: band position (>= 0) or -1 - border index of the two bodies.
// (reductions without a return value: fire-and-forget RED.ADD.F64, no load latency. The storage is zeroed
// first; an entry receives one term per contact between its two bodies -- one for circles --, so the sum does
// not depend on the arrival order unless three or more contacts join the same pair of bodies.)
struct KStore { double *Kb, *KbT, *Brow, *Bcol; int ldk, bw, Nbp; };

__device__ __forceinline__ void k_add(const KStore& c, int ri, int qi, int rj, int qj, double val) {
  if (ri >= 0 && rj >= 0) {
    const int i = 3 * ri + qi, j = 3 * rj + qj;
    if (j <= i) atomicAdd(&c.Kb[(size_t)i * c.ldk + c.bw - (i - j)], val);
    else atomicAdd(&c.KbT[(size_t)j * c.ldk + c.bw - (j - i)], val);
  } else if (ri >= 0) {
    atomicAdd(&c.Brow[(size_t)(3 * ri + qi) * (2 * BD) + BD + 3 * (-1 - rj) + qj], val);
  } else if (rj >= 0) {
    atomicAdd(&c.Brow[(size_t)(3 * rj + qj) * (2 * BD) + 3 * (-1 - ri) + qi], val);
  }
}

// Kb / KbT / Brow / Bcol / Cn <- [[Q + sum_c E_c, A^T], [A, 0]] in the band order
__device__ __noinline__ void assemble_band(const Ctx& c) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int Nbp = c.Nbp, ldk = c.ldk, bw = c.bw;
  {   // zero the arrow storage with 16-byte stores (every array starts 16-byte aligned: bal2 offsets)
    const double2 z2 = make_double2(0.0, 0.0);
    const size_t nk = (size_t)Nbp * ldk, nk2 = nk >> 1, nb2 = (size_t)BD * Nbp;             // interleaved border: 2 BD Nbp doubles
    double2* const k2 = reinterpret_cast<double2*>(c.Kb);
    double2* const kt2 = reinterpret_cast<double2*>(c.KbT);
    for (size_t t = tid; t < nk2; t += NT) { k2[t] = z2; kt2[t] = z2; }
    if ((nk & 1) && tid == 0) { c.Kb[nk - 1] = 0.0; c.KbT[nk - 1] = 0.0; }
    double2* const br2 = reinterpret_cast<double2*>(c.Brow);
    for (size_t t = tid; t < nb2; t += NT) br2[t] = z2;
  }
  for (int t = tid; t < BD * BD; t += NT) c.Cn[t] = (t / BD == t % BD && t / BD >= c.nbd) ? 1.0 : 0.0;
  __syncthreads();
  for (int i = c.Nb + tid; i < Nbp; i += NT) c.Kb[(size_t)i * ldk + bw] = 1.0;      // identity padding
  KStore ks;
  ks.Kb = c.Kb; ks.KbT = c.KbT; ks.Brow = c.Brow; ks.Bcol = c.Bcol; ks.ldk = ldk; ks.bw = bw; ks.Nbp = Nbp;
  const int* const rank = c.rank;
  const int* const start = c.start;
  const int* const adj = c.adj;
  const double* const Eall = c.E;
  // band bodies: one thread per body, its three rows; the diagonal block is summed in registers (list order)
  for (int body = tid; body < c.nb; body += NT) {
    const int rb = rank[body];
    if (rb < 0) continue;
    double dg[9];
#pragma unroll
    for (int u = 0; u < 9; ++u) dg[u] = 0.0;
#pragma unroll
    for (int q = 0; q < 3; ++q) dg[4 * q] = c.qd[3 * body + q];
    const int s0 = start[body], s1 = start[body + 1];
    for (int it = s0; it < s1; ++it) {
      const int a = adj[it], k = a >> 1, side = a & 1;
      const int other = side ? c.b1[k] : c.b2[k];
      const bool two = other < c.nb;                                        // else a static obstacle: diagonal only
      const int ro = two ? rank[other] : 0;
      const double* Eo = Eall + 36 * (size_t)k;
#pragma unroll
      for (int q = 0; q < 3; ++q)
#pragma unroll
        for (int q2 = 0; q2 < 3; ++q2) {
          dg[3 * q + q2] += Eo[(3 * side + q) * 6 + 3 * side + q2];
          if (two) k_add(ks, rb, q, ro, q2, Eo[(3 * side + q) * 6 + 3 * (1 - side) + q2]);
        }
    }
#pragma unroll
    for (int q = 0; q < 3; ++q)
#pragma unroll
      for (int q2 = 0; q2 < 3; ++q2) k_add(ks, rb, q, rb, q2, dg[3 * q + q2]);
  }
  // border bodies: one warp per body, lanes stride over its (long) contact list
  for (int body = warp; body < c.nb; body += NT / 32) {
    const int rb = c.rank[body];
    if (rb >= 0) continue;
    const int bi = -1 - rb;
    double dg[9];
#pragma unroll
    for (int u = 0; u < 9; ++u) dg[u] = 0.0;
    const int s0 = start[body], s1 = start[body + 1];
    for (int it = s0 + lane; it < s1; it += 32) {
      const int a = adj[it], k = a >> 1, side = a & 1;
      const int other = side ? c.b1[k] : c.b2[k];
      const bool two = other < c.nb;                                        // else a static obstacle: diagonal only
      const int ro = two ? rank[other] : 0;
      const double* Eo = Eall + 36 * (size_t)k;
#pragma unroll
      for (int q = 0; q < 3; ++q)
#pragma unroll
        for (int q2 = 0; q2 < 3; ++q2) {
          dg[3 * q + q2] += Eo[(3 * side + q) * 6 + 3 * side + q2];
          const double val = Eo[(3 * side + q) * 6 + 3 * (1 - side) + q2];
          if (!two) continue;
          if (ro >= 0) k_add(ks, rb, q, ro, q2, val);
          else atomicAdd(&c.Cn[(3 * bi + q) * BD + 3 * (-1 - ro) + q2], val);
        }
    }
#pragma unroll
    for (int u = 0; u < 9; ++u) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) dg[u] += __shfl_xor_sync(FULL, dg[u], o);
    }
    if (lane < 9) {
      double val = 0.0;
#pragma unroll
      for (int u = 0; u < 9; ++u) if (lane == u) val = dg[u];
      const int q = lane / 3, q2 = lane - 3 * q;
      if (q == q2) val += c.qd[3 * body + q];
      atomicAdd(&c.Cn[(3 * bi + q) * BD + 3 * bi + q2], val);
    }
  }
  // equality rows: [A 0] / [A^T; 0] inside the corner (their bodies are border bodies)
  for (int t = tid; t < c.e * c.n; t += NT) {
    const double av = c.A[t];
    if (av == 0.0) continue;
    const int k = t / c.n, j = t - k * c.n, body = j / 3, q = j - 3 * body;
    const int bi = -1 - c.rank[body];
    const int row = 3 * c.nbb + k, col = 3 * bi + q;
    c.Cn[row * BD + col] = av;
    c.Cn[col * BD + row] = av;
  }
  __syncthreads();
}

// ------------------------------------------------------------------ arrow-band LU (no pivoting)
// Window: rows / columns k0 .. k0 + Wc - 1 of the band part at slot (i mod Wc), the border at slots Wc ..
// Wc + BD - 1. A pass eliminates the 8 pivots k0 .. k0 + 7: every thread factors the 8 x 8 diagonal block in
// registers (two pivots per reciprocal pair), one thread per panel row / column does the triangular solve
// for its 8 entries, the trailing (bwa + BD)^2 block gets a rank-8 update from the two panels, and the rows /
// columns k0 + Wc .. k0 + Wc + 7 replace the eliminated ones (their global loads are issued before the
// update and stored after it). Factors of pass p go to FB[p] = {D (8x8: L11 \ U11), 1/diag(U11) (8),
// L21^T [8][LP], U12 [8][LP]}, LP = bwa + BD (band rows / columns first, the border at bwa ..).
// Rows / columns entering the window. Warp w owns entering index i = base + w (8 warps = 8 pivots per pass);
// its lanes stride over the band row Kb[i][0..bw] (columns i - bw .. i) and the band column KbT[i][0..bw)
// (rows i - bw .. i - 1), plus the 16 + 16 border entries. Loads and stores are separate steps so that a
// pass can issue the loads before its trailing update and store after it.
constexpr int ER = 5;               // ceil((bw + 1) / 32) for bw <= 159 (bw <= 130 here: bwa <= 128)
struct Entering { double row[ER], col[ER], br; };

__device__ __forceinline__ void enter_load(Entering& en, const double* __restrict__ Kb, const double* __restrict__ KbT,
                                           const double* __restrict__ Brow, const double* __restrict__ Bcol, int i,
                                           int Nbp, int ldk, int bw, int lane) {
  const bool ent = i < Nbp;
#pragma unroll
  for (int q = 0; q < ER; ++q) {
    if (32 * q > bw) break;                                                 // (warp-uniform: rounds beyond the band are skipped)
    const int u = lane + 32 * q;
    en.row[q] = (ent && u <= bw) ? Kb[(size_t)i * ldk + u] : 0.0;
    en.col[q] = (ent && u < bw) ? KbT[(size_t)i * ldk + u] : 0.0;
  }
  en.br = ent ? Brow[(size_t)i * (2 * BD) + lane] : 0.0;                    // interleaved border storage: one line
}

// si: slot of i. Entries with a negative partner index (initial fill) are skipped.
__device__ __forceinline__ void enter_store(const Entering& en, double* win, int i, int si, int lo, int Nbp, int Wc,
                                            int LDW, int bw, int lane) {
  if (i >= Nbp) return;
  int js0 = si + Wc - bw;                       // slot of column i - bw
  if (js0 >= Wc) js0 -= Wc;
#pragma unroll
  for (int q = 0; q < ER; ++q) {
    if (32 * q > bw) break;
    const int u = lane + 32 * q;
    int sj = js0 + u;
    if (sj >= Wc) sj -= Wc;
    if (u <= bw && i - bw + u >= 0) {
      win[si * LDW + sj] = en.row[q];
      if (u < bw) win[sj * LDW + si] = en.col[q];
    }
  }
  // the rest of the slot row / column (partners max(lo, i - Wc + 1) .. i - bw - 1; lo = first index that is
  // still in the window -- the slots below it belong to the other entering rows) is outside the band: zero
  const int nz = Wc - 1 - bw;                   // <= 14
  if (lane < nz && i - Wc + 1 + lane >= lo) {
    int sj = si + 1 + lane;
    if (sj >= Wc) sj -= Wc;
    win[si * LDW + sj] = 0.0;
    win[sj * LDW + si] = 0.0;
  }
  if (lane < BD) win[(Wc + lane) * LDW + si] = en.br;
  else win[si * LDW + Wc + lane - BD] = en.br;
}

// 8 x 8 diagonal block at window slots d0 .. d0 + 7: LU without pivoting in registers (every lane of the calling
// warp redundantly; two pivots per reciprocal pair), published to shared memory for the panel threads:
// dfac[0..63] = L11 \\ U11 row-major, dfac[64..71] = 1 / diag(U11). (16-byte stores: dfac is 16-byte aligned.)
__device__ __forceinline__ void factor_diag(const double* win, int LDW, int d0, double* dfac) {
  double D[8][8], rd[8];
#pragma unroll
  for (int p = 0; p < 8; ++p)
#pragma unroll
    for (int q = 0; q < 8; ++q) D[p][q] = win[(d0 + p) * LDW + d0 + q];
#pragma unroll
  for (int k = 0; k < 8; k += 2) {
    const double r0 = cnd::rcp64_fast(D[k][k]);
    const double r1 = D[k][k] * cnd::rcp64_fast(fma(D[k][k], D[k + 1][k + 1], -(D[k + 1][k] * D[k][k + 1])));
    rd[k] = r0; rd[k + 1] = r1;
#pragma unroll
    for (int i = k + 1; i < 8; ++i) {
      D[i][k] *= r0;
#pragma unroll
      for (int j = k + 1; j < 8; ++j) D[i][j] = fma(-D[i][k], D[k][j], D[i][j]);
    }
#pragma unroll
    for (int i = k + 2; i < 8; ++i) {
      D[i][k + 1] *= r1;
#pragma unroll
      for (int j = k + 2; j < 8; ++j) D[i][j] = fma(-D[i][k + 1], D[k + 1][j], D[i][j]);
    }
  }
  // every lane holds the same values and stores them to the same addresses (one wavefront per store)
  double2* const o = reinterpret_cast<double2*>(dfac);
#pragma unroll
  for (int p = 0; p < 8; ++p)
#pragma unroll
    for (int q = 0; q < 8; q += 2) o[(p * 8 + q) >> 1] = make_double2(D[p][q], D[p][q + 1]);
#pragma unroll
  for (int p = 0; p < 8; p += 2) o[32 + (p >> 1)] = make_double2(rd[p], rd[p + 1]);
}

// -DLCP_BAND_LUPROF (debug build): split the LU time into diag+D-store / panels / entering loads + update /
// entering stores, accumulated into the RESID / STEP / POST / RHS counters (subtract their normal values).
#ifdef LCP_BAND_LUPROF
#define LUPROF_LAP(ph) pf.lap(ph)
#else
#define LUPROF_LAP(ph)
#endif
__device__ __noinline__ void band_lu(const Ctx& c, BProf& pf) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int Wc = c.Wc, LDW = c.LDW, bwa = c.bwa, Nbp = c.Nbp, LP = c.LP, bw = c.bw, ldk = c.ldk, npass = c.npass;
  const int fbs = c.fbs;
  double* const win = smem_d(c.o_win);
  double* const lp = smem_d(c.o_lp);
  double* const up = smem_d(c.o_up);
  double* const FB = c.FB;
  const double* const Kb = c.Kb;
  const double* const KbT = c.KbT;
  const double* const Brow = c.Brow;
  const double* const Bcol = c.Bcol;
  for (int t = tid; t < BD * BD; t += NT) win[(Wc + t / BD) * LDW + Wc + t % BD] = c.Cn[t];
  // initial window: rows / columns 0 .. Wc - 1 enter, eight at a time
  for (int g = 0; g < Wc / PV; ++g) {
    const int i = PV * g + warp;
    Entering en;
    enter_load(en, Kb, KbT, Brow, Bcol, i, Nbp, ldk, bw, lane);
    enter_store(en, win, i, i, 0, Nbp, Wc, LDW, bw, lane);
  }
  __syncthreads();
  if (warp == 0) factor_diag(win, LDW, 0, smem_d(c.o_cf));
  __syncthreads();
  int s0 = 0;                                                               // slot of pivot k0
  for (int ps = 0; ps < npass; ++ps) {
    const int k0 = PV * ps;
    const int na = min(bwa, Nbp - (k0 + PV));
    const int Lr = na + BD;
    double* const fb = FB + (size_t)ps * fbs;
    // ---- 8 x 8 diagonal block: dfac[ps & 1] was factored by warp 0 during the previous pass (look-ahead, see the
    // update phase below); warp 1 copies it to the factor block
    double* const dfac = smem_d(c.o_cf) + 72 * (ps & 1);                    // (the corner factors land here only after the last pass)
    if (warp == 1)
      for (int i = lane; i < 72; i += 32) {                                   // the substitutions' copy: U11 rows scaled by 1 / u_pp
        const int p = i >> 3, q = i & 7;
        fb[i] = (i < 64 && q > p) ? dfac[i] * dfac[64 + p] : dfac[i];
      }
    LUPROF_LAP(BPH_RESID);
    // ---- panels: rows of L21 (t < Lr), columns of U12 (Lr <= t < 2 Lr)
    for (int t = tid; t < 2 * Lr; t += NT) {
      const bool isrow = t < Lr;
      const int rel = isrow ? t : t - Lr;
      int slot, pr;                                                         // window slot, panel index
      if (rel < na) { slot = s0 + PV + rel; if (slot >= Wc) slot -= Wc; pr = rel; }
      else { slot = Wc + rel - na; pr = bwa + rel - na; }
      double a[8];
      if (isrow) {
#pragma unroll
        for (int q = 0; q < 8; ++q) a[q] = win[slot * LDW + s0 + q];
#pragma unroll
        for (int q = 0; q < 8; ++q) {                                       // x U11 = a
#pragma unroll
          for (int p = 0; p < q; ++p) a[q] = fma(-a[p], dfac[p * 8 + q], a[q]);
          a[q] *= dfac[64 + q];
        }
#pragma unroll
        for (int q = 0; q < 8; ++q) { lp[pr * 8 + q] = a[q]; fb[72 + q * LP + pr] = a[q]; }
      } else {
#pragma unroll
        for (int p = 0; p < 8; ++p) a[p] = win[(s0 + p) * LDW + slot];
#pragma unroll
        for (int p = 1; p < 8; ++p)                                         // L11 y = a
#pragma unroll
          for (int q = 0; q < p; ++q) a[p] = fma(-dfac[p * 8 + q], a[q], a[p]);
#pragma unroll
        for (int p = 0; p < 8; ++p) { up[p * LP + pr] = a[p]; fb[72 + 8 * LP + p * LP + pr] = a[p]; }
      }
    }
    __syncthreads();
    LUPROF_LAP(BPH_STEP);
    // ---- entering row / column of this warp: loads now, stores after the update
    Entering en;
    enter_load(en, Kb, KbT, Brow, Bcol, k0 + Wc + warp, Nbp, ldk, bw, lane);
    LUPROF_LAP(BPH_WINV);
    // ---- trailing update C -= L21 U12 (rank 8) on the FP64 tensor pipe: the (na + BD)^2 region is cut into
    // 8 x 8 tiles (a tile's 8 rows / columns are consecutive window slots: s0, Wc and na are multiples of 8, so a
    // tile never wraps), a warp takes half tile rows and issues two mma.sync.m8n8k4.f64 per tile
    // (k = pivots 0-3, 4-7) with A = -L21 (lp, [row][8]) and B = U12 (up, [8][LP]). Fragments (PTX ISA, m8n8k4):
    // A: lane holds (row g, k t), B: (k t, column g), C/D: (row g, columns 2t, 2t + 1), g = lane / 4, t = lane % 4.
    // One DMMA carries 256 FMAs: 242 instructions per pass instead of 3872 DFMAs, at the same FP64 datapath rate
    // (measured: 8 warps reach 92 % of the DMMA peak, 54 % of the DFMA peak; profiles/r02_ubench_pipes_latencies.txt).
    {
      const int g = lane >> 2, t = lane & 3;
      const int ntb = na >> 3, ntl = ntb + BD / 8;                          // band tiles, all tiles per dimension
      const int hc = (ntl + 1) >> 1;
      // Look-ahead: warp 0 updates tile (0, 0) -- the NEXT diagonal block -- alone, factors it (a serial chain of
      // ~2000 cycles) and publishes it for the next pass while warps 1..7 do the other tiles.
      // Work unit of those = half a tile row (2 ntl units); no division, the A fragments stay in registers.
      if (warp == 0) {
        if (ps + 1 < npass) {
          int d0 = s0 + PV; if (d0 >= Wc) d0 -= Wc;
          const double a0 = -lp[g * 8 + t], a1 = -lp[g * 8 + 4 + t];
          const double b0 = up[t * LP + g], b1 = up[(4 + t) * LP + g];
          double* const cptr = win + (d0 + g) * LDW + d0 + 2 * t;
          double c0 = cptr[0], c1 = cptr[1];
          asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
              : "+d"(c0), "+d"(c1) : "d"(a0), "d"(b0));
          asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
              : "+d"(c0), "+d"(c1) : "d"(a1), "d"(b1));
          cptr[0] = c0; cptr[1] = c1;
          __syncwarp();
          factor_diag(win, LDW, d0, smem_d(c.o_cf) + 72 * ((ps + 1) & 1));
        }
      } else
      for (int w = warp - 1; w < 2 * ntl; w += NT / 32 - 1) {
        const int R = w >> 1;
        const int c_lo = (w & 1) ? hc : ((R == 0 && ps + 1 < npass) ? 1 : 0), c_hi = (w & 1) ? ntl : hc;   // tile (0, 0) is warp 0's
        int rslot0, rpr0;
        if (R < ntb) { rslot0 = s0 + PV + 8 * R; if (rslot0 >= Wc) rslot0 -= Wc; rpr0 = 8 * R; }
        else { rslot0 = Wc + 8 * (R - ntb); rpr0 = bwa + 8 * (R - ntb); }
        const double a0 = -lp[(rpr0 + g) * 8 + t], a1 = -lp[(rpr0 + g) * 8 + 4 + t];
        double* const crow = win + (rslot0 + g) * LDW + 2 * t;
        const double* const ub0 = up + t * LP + g;
        const double* const ub1 = up + (4 + t) * LP + g;
        // TB tiles in flight: all operand loads, then the 2 TB DMMAs, then the stores (a tile alone is a serial
        // chain LDS -> DMMA -> DMMA -> STS of ~200 cycles, and 8 warps do not hide it)
        constexpr int TB = 3;
        for (int Cb0 = c_lo; Cb0 < c_hi; Cb0 += TB) {
          double* cptr[TB];
          double c0[TB], c1[TB], b0[TB], b1[TB];
          bool live[TB];
#pragma unroll
          for (int u = 0; u < TB; ++u) {
            live[u] = Cb0 + u < c_hi;
            const int Cb = live[u] ? Cb0 + u : Cb0;
            int cslot0, cpr0;
            if (Cb < ntb) { cslot0 = s0 + PV + 8 * Cb; if (cslot0 >= Wc) cslot0 -= Wc; cpr0 = 8 * Cb; }
            else { cslot0 = Wc + 8 * (Cb - ntb); cpr0 = bwa + 8 * (Cb - ntb); }
            cptr[u] = crow + cslot0;
            c0[u] = cptr[u][0]; c1[u] = cptr[u][1];
            b0[u] = ub0[cpr0]; b1[u] = ub1[cpr0];
          }
#pragma unroll
          for (int u = 0; u < TB; ++u)
            asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                : "+d"(c0[u]), "+d"(c1[u]) : "d"(a0), "d"(b0[u]));
#pragma unroll
          for (int u = 0; u < TB; ++u)
            asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                : "+d"(c0[u]), "+d"(c1[u]) : "d"(a1), "d"(b1[u]));
#pragma unroll
          for (int u = 0; u < TB; ++u)
            if (live[u]) { cptr[u][0] = c0[u]; cptr[u][1] = c1[u]; }
        }
      }
    }
    LUPROF_LAP(BPH_POST);
    enter_store(en, win, k0 + Wc + warp, s0 + warp, k0 + PV, Nbp, Wc, LDW, bw, lane);
    __syncthreads();
    LUPROF_LAP(BPH_RHS);
    s0 += PV;
    if (s0 >= Wc) s0 -= Wc;
  }
  // ---- corner: dense LU of the 16 x 16 border block
  {
    const int i = tid >> 4, j = tid & 15;
    double* cn = win + Wc * LDW + Wc;
    for (int k = 0; k < BD; ++k) {
      if (j == k && i > k) cn[i * LDW + k] /= cn[k * LDW + k];
      __syncthreads();
      if (i > k && j > k) cn[i * LDW + j] = fma(-cn[i * LDW + k], cn[k * LDW + j], cn[i * LDW + j]);
      __syncthreads();
    }
    smem_d(c.o_cf)[tid] = cn[i * LDW + j];
    __syncthreads();
  }
}

// ------------------------------------------------------------------ substitution: sol <- Kbar^-1 sol
// Warp 0 solves, pass by pass, from a chunk of factor blocks in shared memory; the other warps fetch the
// next chunk from the L2 workspace into the other half of the (idle) window region.
// (cp.async: the copies are in flight together, no register staging; the caller's __syncthreads publishes them)
__device__ __forceinline__ void fetch_chunk(const double* FB, int fbs, double* dst, int p_lo, int p_hi, int t, int nt) {
  const int cnt2 = (p_hi - p_lo) * (fbs >> 1);                              // fbs is even: 16-byte copies
  const double2* src = reinterpret_cast<const double2*>(FB + (size_t)p_lo * fbs);
  const unsigned d0 = (unsigned)__cvta_generic_to_shared(dst);
  for (int i = t; i < cnt2; i += nt)
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d0 + 16u * (unsigned)i), "l"(src + i) : "memory");
  asm volatile("cp.async.wait_all;" ::: "memory");
}

struct SolveDims { double* sol; int bwa, Nbp, LP; };

// One substitution pass is a latency chain on one warp (8 pivots, then the rows they touch), so the row updates
// are fully unrolled (SUBR rounds of 32 rows + the border, predicated: all chains in flight together) instead of
// a loop whose iterations each wait for LDS -> 8 dependent DFMAs -> STS.
constexpr int SUBR = 4;             // ceil(max bwa / 32); carve_bplan caps bwa at 32 SUBR

__device__ __forceinline__ void pass_forward(const SolveDims c, const double* blk, int ps, int lane) {
  const int k0 = PV * ps, na = min(c.bwa, c.Nbp - (k0 + PV)), LP = c.LP;
  double y[8];
#pragma unroll
  for (int p = 0; p < 8; ++p) y[p] = c.sol[k0 + p];
  const double* L = blk + 72;
  int relc[SUBR];
  bool ok[SUBR];
  double acc[SUBR];
#pragma unroll
  for (int r = 0; r < SUBR; ++r) {
    const int rel = lane + 32 * r;
    ok[r] = rel < na;
    relc[r] = ok[r] ? rel : 0;
    acc[r] = c.sol[k0 + PV + relc[r]];
  }
  const bool okb = lane < BD;
  const int lb = c.bwa + (okb ? lane : 0);
  double accb = c.sol[c.Nbp + (okb ? lane : 0)];
#pragma unroll
  for (int p = 1; p < 8; ++p)
#pragma unroll
    for (int q = 0; q < p; ++q) y[p] = fma(-blk[p * 8 + q], y[q], y[p]);
  __syncwarp();                                                             // every lane has read sol[k0 ..] before lane 0 overwrites it
  if (lane == 0) {
#pragma unroll
    for (int p = 0; p < 8; ++p) c.sol[k0 + p] = y[p];
  }
#pragma unroll
  for (int p = 0; p < 8; ++p) {
#pragma unroll
    for (int r = 0; r < SUBR; ++r) acc[r] = fma(-L[p * LP + relc[r]], y[p], acc[r]);
    accb = fma(-L[p * LP + lb], y[p], accb);
  }
#pragma unroll
  for (int r = 0; r < SUBR; ++r)
    if (ok[r]) c.sol[k0 + PV + relc[r]] = acc[r];
  if (okb) c.sol[c.Nbp + lane] = accb;
  __syncwarp();
}

// blk[p * 8 + q], q > p, holds U11[p][q] / U11[p][p] (scaled when the factor block is written), so that the
// 8-pivot chain is one FMA per step: x_p = (b_p - tail_p) / u_pp - sum_{q > p} (u_pq / u_pp) x_q.
__device__ __forceinline__ void pass_backward(const SolveDims c, const double* blk, int ps, int lane) {
  const int k0 = PV * ps, na = min(c.bwa, c.Nbp - (k0 + PV)), LP = c.LP;
  const double* U = blk + 72 + 8 * LP;
  double acc[8];
#pragma unroll
  for (int p = 0; p < 8; ++p) acc[p] = 0.0;
#pragma unroll
  for (int r = 0; r < SUBR; ++r) {
    const int rel = lane + 32 * r;
    const bool ok = rel < na;
    const int rc = ok ? rel : 0;
    const double xv = ok ? c.sol[k0 + PV + rc] : 0.0;
    // a select, not a product with xv = 0: in the last pass (na = 0) panel entry 0 is never written
#pragma unroll
    for (int p = 0; p < 8; ++p) acc[p] = ok ? fma(U[p * LP + rc], xv, acc[p]) : acc[p];
  }
  {
    const bool okb = lane < BD;
    const int lb = okb ? lane : 0;
    const double xv = okb ? c.sol[c.Nbp + lb] : 0.0;
#pragma unroll
    for (int p = 0; p < 8; ++p) acc[p] = fma(U[p * LP + c.bwa + lb], xv, acc[p]);
  }
  // 8 sums over 32 lanes: halve the number of values per lane at every butterfly stage (9 exchanges instead of
  // 40); lane l ends with the total of p = 4 b16 + 2 b8 + b4 (bits of l), then the 8 totals are broadcast
  double v4[4], v2[2], v1;
  {
    const bool hi = lane & 16;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const double send = hi ? acc[j] : acc[j + 4], keep = hi ? acc[j + 4] : acc[j];
      v4[j] = keep + __shfl_xor_sync(FULL, send, 16);
    }
  }
  {
    const bool hi = lane & 8;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const double send = hi ? v4[j] : v4[j + 2], keep = hi ? v4[j + 2] : v4[j];
      v2[j] = keep + __shfl_xor_sync(FULL, send, 8);
    }
  }
  {
    const bool hi = lane & 4;
    const double send = hi ? v2[0] : v2[1], keep = hi ? v2[1] : v2[0];
    v1 = keep + __shfl_xor_sync(FULL, send, 4);
  }
  v1 += __shfl_xor_sync(FULL, v1, 2);
  v1 += __shfl_xor_sync(FULL, v1, 1);
  double x[8];
#pragma unroll
  for (int p = 0; p < 8; ++p) {
    const double tot = __shfl_sync(FULL, v1, 16 * ((p >> 2) & 1) + 8 * ((p >> 1) & 1) + 4 * (p & 1));
    x[p] = (c.sol[k0 + p] - tot) * blk[64 + p];
  }
#pragma unroll
  for (int p = 6; p >= 0; --p)
#pragma unroll
    for (int q = p + 1; q < 8; ++q) x[p] = fma(-blk[p * 8 + q], x[q], x[p]);
  __syncwarp();                                                             // (same: reads of sol[k0 ..] before the overwrite)
  if (lane == 0) {
#pragma unroll
    for (int p = 0; p < 8; ++p) c.sol[k0 + p] = x[p];
  }
  __syncwarp();
}

__device__ __noinline__ void band_solve(const Ctx& c) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int npass = c.npass, fbs = c.fbs;
  const double* const FB = c.FB;
  SolveDims sd;
  sd.sol = smem_d(c.o_sol); sd.bwa = c.bwa; sd.Nbp = c.Nbp; sd.LP = c.LP;
  const int CH = max(1, min(npass, (c.win_doubles / 2) / fbs));             // passes per chunk
  const int nch = (npass + CH - 1) / CH;
  double* const buf0 = smem_d(c.o_win);
  double* const buf1 = buf0 + (size_t)CH * fbs;
  // ---- forward
  fetch_chunk(FB, fbs, buf0, 0, min(CH, npass), tid, NT);
  __syncthreads();
  for (int ch = 0; ch < nch; ++ch) {
    if (warp == 0) {
      const int p_lo = ch * CH, p_hi = min(npass, p_lo + CH);
      for (int ps = p_lo; ps < p_hi; ++ps) pass_forward(sd, ((ch & 1) ? buf1 : buf0) + (size_t)(ps - p_lo) * fbs, ps, lane);
    } else if (ch + 1 < nch) {
      fetch_chunk(FB, fbs, ((ch + 1) & 1) ? buf1 : buf0, (ch + 1) * CH, min(npass, (ch + 2) * CH), tid - 32, NT - 32);
    }
    __syncthreads();
  }
  // ---- corner (16 x 16 dense factors) ; meanwhile the last chunk is already resident for the way back
  if (warp == 0) {
    const double* const cf = smem_d(c.o_cf);
    double* const solb = sd.sol + c.Nbp;
    double yi = lane < BD ? solb[lane] : 0.0;
    const int li = lane < BD ? lane : 0;
    for (int k = 0; k < BD; ++k) {
      const double yk = __shfl_sync(FULL, yi, k);
      if (lane < BD && lane > k) yi = fma(-cf[li * BD + k], yk, yi);
    }
    for (int k = BD - 1; k >= 0; --k) {
      if (lane == k) yi /= cf[k * BD + k];
      const double xk = __shfl_sync(FULL, yi, k);
      if (lane < k) yi = fma(-cf[li * BD + k], xk, yi);
    }
    if (lane < BD) solb[lane] = yi;
  }
  __syncthreads();
  // ---- backward (chunk nch - 1 sits in buf[(nch - 1) & 1])
  for (int ch = nch - 1; ch >= 0; --ch) {
    if (warp == 0) {
      const int p_lo = ch * CH, p_hi = min(npass, p_lo + CH);
      for (int ps = p_hi - 1; ps >= p_lo; --ps) pass_backward(sd, ((ch & 1) ? buf1 : buf0) + (size_t)(ps - p_lo) * fbs, ps, lane);
    } else if (ch > 0) {
      fetch_chunk(FB, fbs, ((ch - 1) & 1) ? buf1 : buf0, (ch - 1) * CH, ch * CH, tid - 32, NT - 32);
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------ solve_kkt (pdipm.py:325-354)
// rx[n], rs[m], rz[m], ry[e] (nullptr = 0)  ->  dx[n], ds[m], dz[m], dy[e].  dz may alias rs.
__device__ __forceinline__ void contact_t(const Ctx& c, int k, const double* rs, const double* rz, double (&t)[4]) {
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    t[r] = 0.0;
    if (r < c.cs) { const int i = r * c.ncap + k; t[r] = (rz ? rz[i] : 0.0) - rs[i] / c.d[i]; }
  }
}

__device__ __forceinline__ void apply_W(const Ctx& c, int k, const double (&t)[4], double (&v)[4]) {
  const double* Wk = c.W + 16 * (size_t)k;
  if (c.cs == 1) { v[0] = Wk[0] * t[0]; v[1] = v[2] = v[3] = 0.0; return; }
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    double a = 0.0;
#pragma unroll
    for (int q = 0; q < 4; ++q) a = fma(Wk[r * 4 + q], t[q], a);
    v[r] = a;
  }
}

__device__ __noinline__ void solve_kkt(const Ctx& c, BProf& pf, const double* rx, const double* rs, const double* rz,
                                       const double* ry, double* dx, double* ds, double* dz, double* dy) {
  const int tid = threadIdx.x, ncap = c.ncap;
  // v = W (rz - rs/d), kept as (v_n, v_f1 - v_f2) per contact in c.t
  for (int k = tid; k < c.nc; k += NT) {
    double t[4], v[4];
    contact_t(c, k, rs, rz, t);
    apply_W(c, k, t, v);
    c.t[k] = v[0];
    if (c.cs == 4) c.t[ncap + k] = v[1] - v[2];
  }
  for (int i = tid; i < c.Nbp + BD; i += NT) c.sol[i] = 0.0;
  __syncthreads();
  for (int body = tid; body < c.nb; body += NT) {                            // rhs = -rx - G^T v
    double acc[3] = {0.0, 0.0, 0.0};
    const int s0 = c.start[body], s1 = c.start[body + 1];
    for (int it = s0; it < s1; ++it) {
      const int a = c.adj[it], k = a >> 1, side = a & 1;
      const double* g = c.cg + 12 * (size_t)k + 3 * side;
      const double vn = c.t[k], vf = c.cs == 4 ? c.t[ncap + k] : 0.0;
#pragma unroll
      for (int q = 0; q < 3; ++q) acc[q] = fma(g[q], vn, acc[q]);
      if (c.cs == 4) {
#pragma unroll
        for (int q = 0; q < 3; ++q) acc[q] = fma(g[6 + q], vf, acc[q]);
      }
    }
#pragma unroll
    for (int q = 0; q < 3; ++q) c.sol[sol_index(c, body, q)] = -(rx ? rx[3 * body + q] : 0.0) - acc[q];
  }
  for (int k = tid; k < c.e; k += NT) c.sol[c.Nbp + 3 * c.nbb + k] = -(ry ? ry[k] : 0.0);
  __syncthreads();
  pf.lap(BPH_RHS);
  band_solve(c);
  pf.lap(BPH_SUBST);
  for (int k = tid; k < c.nc; k += NT) {                                    // dz = W (G dx + t), ds = (-rs - dz)/d
    double t[4], v[4];
    contact_t(c, k, rs, rz, t);
    const double* g = c.cg + 12 * (size_t)k;
    const int b1 = c.b1[k], b2 = c.b2[k];
    double x1[3], x2[3];
#pragma unroll
    for (int q = 0; q < 3; ++q) { x1[q] = c.sol[sol_index(c, b1, q)]; x2[q] = b2 < c.nb ? c.sol[sol_index(c, b2, q)] : 0.0; }
    double gn = 0.0, gf = 0.0;
#pragma unroll
    for (int q = 0; q < 3; ++q) { gn = fma(g[q], x1[q], gn); gn = fma(g[3 + q], x2[q], gn); }
    t[0] += gn;
    if (c.cs == 4) {
#pragma unroll
      for (int q = 0; q < 3; ++q) { gf = fma(g[6 + q], x1[q], gf); gf = fma(g[9 + q], x2[q], gf); }
      t[1] += gf; t[2] -= gf;
    }
    apply_W(c, k, t, v);
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      if (r < c.cs) {
        const int i = r * ncap + k;
        const double rsi = rs[i];
        dz[i] = v[r];                                                       // :351
        ds[i] = (-rsi - v[r]) / c.d[i];                                     // :347,350
      }
    }
  }
  for (int body = tid; body < c.nb; body += NT)
#pragma unroll
    for (int q = 0; q < 3; ++q) dx[3 * body + q] = c.sol[sol_index(c, body, q)];
  for (int k = tid; k < c.e; k += NT) dy[k] = c.sol[c.Nbp + 3 * c.nbb + k];
  __syncthreads();
  pf.lap(BPH_POST);
}

// trans: factor K^T (exact-adjoint backward); the forward passes a constant false
__device__ __forceinline__ void factor_kkt(const Ctx& c, BProf& pf, int mode, const double* mu, bool trans) {
  contact_blocks(c, mode, mu, trans);
  __syncthreads();
  pf.lap(BPH_WINV);
  assemble_band(c);
  pf.lap(BPH_ASSEMBLE);
  band_lu(c, pf);
  pf.lap(BPH_LU);
}

// get_step (pdipm.py:182-186) over the rows of this scene (slot-major storage: row r of contact k at r ncap + k)
__device__ __forceinline__ void get_steps(const Ctx& c, const double* z, const double* dz, const double* s,
                                          const double* ds, double& step_z, double& step_s) {
  const double NEG_INF = -INFINITY, POS_INF = INFINITY;
  double mx[2] = {NEG_INF, NEG_INF}, mn[2] = {POS_INF, POS_INF}, any[2] = {0.0, 0.0};
  for (int r = 0; r < c.cs; ++r)
    for (int k = threadIdx.x; k < c.nc; k += NT) {
      const int i = r * c.ncap + k;
      const double az = -z[i] / dz[i], as = -s[i] / ds[i];
      mx[0] = nan_max(mx[0], az);
      mx[1] = nan_max(mx[1], as);
      if (dz[i] > 0.0) any[0] = 1.0; else mn[0] = nan_min(mn[0], az);
      if (ds[i] > 0.0) any[1] = 1.0; else mn[1] = nan_min(mn[1], as);
    }
  double v[6] = {mx[0], mx[1], -mn[0], -mn[1], any[0], any[1]};
  block_reduce<double, 6>(v, OpMax(), NEG_INF, c.red);
  const double fz = (v[0] > 1.0) ? v[0] : 1.0;
  const double fs = (v[1] > 1.0) ? v[1] : 1.0;
  step_z = (v[4] > 0.0) ? nan_min(-v[2], fz) : -v[2];
  step_s = (v[5] > 0.0) ? nan_min(-v[3], fs) : -v[3];
}

// row of lam / slack (reference order for a scene with nc contacts: normal [0,nc), friction [nc,3nc), gamma [3nc,4nc))
__device__ __forceinline__ int out_row(int r, int k, int nc) {
  return r == 0 ? k : (r == 3 ? 3 * nc + k : nc + 2 * k + (r - 1));
}

// ------------------------------------------------------------------ forward (pdipm.py:49-179), one scene
__device__ __forceinline__ void forward_scene(const BArgs& a, Ctx& c, BProf& pf, int sc) {
  const int tid = threadIdx.x, n = c.n, e = c.e, nc = c.nc, cs = c.cs, ncap = c.ncap, m = c.m;
  const int mode = a.soa.mode;
  const double* mu = a.soa.mu ? a.soa.mu + (size_t)sc * a.soa.nc : nullptr;
  const double* b = e > 0 ? a.b + (size_t)sc * e : nullptr;
  double* o_x = a.zhat + (size_t)sc * n;
  double* o_z = a.lam + (size_t)sc * a.P.m;
  double* o_s = a.slack + (size_t)sc * a.P.m;
  double* o_y = e > 0 ? a.nu + (size_t)sc * e : nullptr;
  const int mrows = cs * ncap;
  // ---- initial point: d = 1, rhs (p, 0, -h, -b)                 :58-63
  for (int i = tid; i < mrows; i += NT) { c.d[i] = 1.0; c.rs[i] = 0.0; c.rz[i] = -c.h[i]; }
  for (int i = tid; i < n; i += NT) c.rx[i] = c.ps[i];
  for (int i = tid; i < e; i += NT) c.ry[i] = -b[i];
  __syncthreads();
  factor_kkt(c, pf, mode, mu, false);
  solve_kkt(c, pf, c.rx, c.rs, c.rz, e > 0 ? c.ry : nullptr, c.x, c.s, c.z, c.y);
  pf.count(BPH_FACTORS);
  pf.count(BPH_SOLVES);
  if (m == 0) {                                                             // no contacts: engines.py:35-49
    for (int i = tid; i < n; i += NT) o_x[i] = c.x[i];
    for (int i = tid; i < e; i += NT) o_y[i] = c.y[i];
    if (tid == 0) { a.status[sc] = 2; a.iters[sc] = 0; if (a.resid) a.resid[sc] = 0.0; }
    return;
  }
  {   // shift s and z to >= 1 where the minimum is <= 0          :65-75
    double mn[2] = {INFINITY, INFINITY};
    for (int r = 0; r < cs; ++r)
      for (int k = tid; k < nc; k += NT) { mn[0] = nan_min(mn[0], c.s[r * ncap + k]); mn[1] = nan_min(mn[1], c.z[r * ncap + k]); }
    block_reduce<double, 2>(mn, OpMin(), (double)INFINITY, c.red);
    for (int r = 0; r < cs; ++r)
      for (int k = tid; k < nc; k += NT) {
        if (mn[0] <= 0.0) c.s[r * ncap + k] -= mn[0] - 1.0;
        if (mn[1] <= 0.0) c.z[r * ncap + k] -= mn[1] - 1.0;
      }
    __syncthreads();
  }
  double best = nan("");
  bool have_best = false;
  int not_improved = 0, status = 0, it = 0;
  for (it = 0; it < a.max_iter; ++it) {
    // ---- residuals                                              :82-96
    for (int body = tid; body < c.nb; body += NT) {                          // rx = G^T z + Q x + p (+ A^T y)
      double acc[3] = {0.0, 0.0, 0.0};
      const int s0 = c.start[body], s1 = c.start[body + 1];
      for (int it2 = s0; it2 < s1; ++it2) {
        const int ad = c.adj[it2], k = ad >> 1, side = ad & 1;
        const double* g = c.cg + 12 * (size_t)k + 3 * side;
        const double zn = c.z[k];
#pragma unroll
        for (int q = 0; q < 3; ++q) acc[q] = fma(g[q], zn, acc[q]);
        if (cs == 4) {
          const double zf = c.z[ncap + k] - c.z[2 * ncap + k];
#pragma unroll
          for (int q = 0; q < 3; ++q) acc[q] = fma(g[6 + q], zf, acc[q]);
        }
      }
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const int j = 3 * body + q;
        double t = acc[q];
        for (int k = 0; k < e; ++k) t = fma(c.A[k * n + j], c.y[k], t);
        c.rx[j] = t + c.qd[j] * c.x[j] + c.ps[j];
      }
    }
    for (int k = tid; k < nc; k += NT) {                                    // rz = G x + s - h - F z
      const double* g = c.cg + 12 * (size_t)k;
      const int b1 = c.b1[k], b2 = c.b2[k];
      const bool two = b2 < c.nb;                                          // else a static obstacle: g[3..5], g[9..11] = 0
      const int j2 = two ? 3 * b2 : 3 * b1;
      double gn = 0.0, gf = 0.0;
#pragma unroll
      for (int q = 0; q < 3; ++q) { gn = fma(g[q], c.x[3 * b1 + q], gn); gn = fma(g[3 + q], c.x[j2 + q], gn); }
      if (cs == 4) {
#pragma unroll
        for (int q = 0; q < 3; ++q) { gf = fma(g[6 + q], c.x[3 * b1 + q], gf); gf = fma(g[9 + q], c.x[j2 + q], gf); }
        const double zn = c.z[k], z1 = c.z[ncap + k], z2 = c.z[2 * ncap + k], zg = c.z[3 * ncap + k];
        c.rz[k] = gn + c.s[k] - c.h[k];                                      // F row 0 = 0
        c.rz[ncap + k] = gf + c.s[ncap + k] - c.h[ncap + k] - zg;            // F rows f1, f2: E gamma
        c.rz[2 * ncap + k] = -gf + c.s[2 * ncap + k] - c.h[2 * ncap + k] - zg;
        c.rz[3 * ncap + k] = c.s[3 * ncap + k] - c.h[3 * ncap + k] - (mu[k] * zn - z1 - z2);
      } else {
        c.rz[k] = gn + c.s[k] - c.h[k];
      }
    }
    for (int k = tid; k < e; k += NT) {                                     // ry = A x - b
      double acc = 0.0;
      for (int j = 0; j < n; ++j) acc = fma(c.A[k * n + j], c.x[j], acc);
      c.ry[k] = acc - b[k];
    }
    __syncthreads();
    double q4[4] = {0, 0, 0, 0};                                            // s.z, |rz|^2, |ry|^2, |rx|^2
    for (int r = 0; r < cs; ++r)
      for (int k = tid; k < nc; k += NT) { const int i = r * ncap + k; q4[0] += c.s[i] * c.z[i]; q4[1] += c.rz[i] * c.rz[i]; }
    for (int i = tid; i < e; i += NT) q4[2] += c.ry[i] * c.ry[i];
    for (int i = tid; i < n; i += NT) q4[3] += c.rx[i] * c.rx[i];
    block_reduce<double, 4>(q4, OpSum(), 0.0, c.red);
    pf.lap(BPH_RESID);
    const double sz = q4[0];
    const double mu_ = fabs(sz / (double)m);                                // :91
    const double resid = (e > 0 ? sqrt(q4[2]) : 0.0) + sqrt(q4[1]) + sqrt(q4[3]) + (double)m * mu_;   // :92-96
    // ---- best iterate / termination                             :107-136
    bool improved;
    if (!have_best) { improved = true; have_best = true; not_improved = 0; }
    else { improved = resid < best; not_improved = improved ? 0 : not_improved + 1; }
    if (improved) {
      best = resid;
      for (int i = tid; i < n; i += NT) o_x[i] = c.x[i];
      for (int r = 0; r < cs; ++r)
        for (int k = tid; k < nc; k += NT) { const int o = out_row(r, k, nc); o_z[o] = c.z[r * ncap + k]; o_s[o] = c.s[r * ncap + k]; }
      for (int i = tid; i < e; i += NT) o_y[i] = c.y[i];
    }
    if (not_improved == a.not_improved_lim) { status = 1; ++it; break; }
    if (best < a.eps) { status = 2; ++it; break; }
    if (mu_ > 1e100) { status = 3; ++it; break; }
    if (it + 1 == a.max_iter) { ++it; break; }                              // the step would never be read
    for (int r = 0; r < cs; ++r)
      for (int k = tid; k < nc; k += NT) { const int i = r * ncap + k; c.d[i] = c.z[i] / c.s[i]; }     // :98
    __syncthreads();
    factor_kkt(c, pf, mode, mu, false);                                     // :100
    // ---- affine direction                                       :138-139   (rs = z)
    solve_kkt(c, pf, c.rx, c.z, c.rz, e > 0 ? c.ry : nullptr, c.dx, c.ds, c.dz, c.dy);
    double stz, sts;
    get_steps(c, c.z, c.dz, c.s, c.ds, stz, sts);
    const double alpha_aff = nan_min(nan_min(stz, sts), 1.0);               // :142-144
    double t3[1] = {0.0};
    for (int r = 0; r < cs; ++r)
      for (int k = tid; k < nc; k += NT) { const int i = r * ncap + k; t3[0] += (c.s[i] + alpha_aff * c.ds[i]) * (c.z[i] + alpha_aff * c.dz[i]); }
    block_reduce<double, 1>(t3, OpSum(), 0.0, c.red);
    const double ratio = t3[0] / sz;                                        // :146-150
    const double sig = ratio * ratio * ratio;
    const double musig = -mu_ * sig;                                        // :152-158
    for (int r = 0; r < cs; ++r)
      for (int k = tid; k < nc; k += NT) { const int i = r * ncap + k; c.rs[i] = (musig + c.ds[i] * c.dz[i]) / c.s[i]; }
    __syncthreads();
    pf.lap(BPH_STEP);
    // corrector: dx_c -> rx, ds_c -> rz, dz_c -> rs, dy_c -> ry (dead until the next residual phase)
    solve_kkt(c, pf, nullptr, c.rs, nullptr, nullptr, c.rx, c.rz, c.rs, c.ry);
    for (int i = tid; i < n; i += NT) c.dx[i] += c.rx[i];                   // :160-163
    for (int r = 0; r < cs; ++r)
      for (int k = tid; k < nc; k += NT) { const int i = r * ncap + k; c.ds[i] += c.rz[i]; c.dz[i] += c.rs[i]; }
    for (int i = tid; i < e; i += NT) c.dy[i] += c.ry[i];
    __syncthreads();
    get_steps(c, c.z, c.dz, c.s, c.ds, stz, sts);
    const double alpha = nan_min(0.999 * nan_min(stz, sts), 1.0);           // :164-166
    for (int i = tid; i < n; i += NT) c.x[i] += alpha * c.dx[i];            // :171-174
    for (int r = 0; r < cs; ++r)
      for (int k = tid; k < nc; k += NT) { const int i = r * ncap + k; c.s[i] += alpha * c.ds[i]; c.z[i] += alpha * c.dz[i]; }
    for (int i = tid; i < e; i += NT) c.y[i] += alpha * c.dy[i];
    __syncthreads();
    pf.lap(BPH_STEP);
    pf.count(BPH_FACTORS);
    pf.count(BPH_SOLVES, 2);
  }
  if (tid == 0) { a.status[sc] = status; a.iters[sc] = it; if (a.resid) a.resid[sc] = best; }
}

__device__ __forceinline__ void init_ctx(Ctx& c, const BPlan& P, double* wsd, int* wsi) {
  c.red = reinterpret_cast<double*>(bnd_smem + P.o_red);
  c.sv = reinterpret_cast<int*>(bnd_smem + P.o_sv);
  c.rank = reinterpret_cast<int*>(bnd_smem + P.o_rank);
  c.cf = reinterpret_cast<double*>(bnd_smem + P.o_cf);
  c.sol = reinterpret_cast<double*>(bnd_smem + P.o_sol);
  c.lp = reinterpret_cast<double*>(bnd_smem + P.o_lp);
  c.up = reinterpret_cast<double*>(bnd_smem + P.o_up);
  c.win = reinterpret_cast<double*>(bnd_smem + P.o_win);
  c.win_doubles = P.win_bytes / 8;
  c.bwa_max = P.bwa_max;
  c.o_win = P.o_win; c.o_sol = P.o_sol; c.o_lp = P.o_lp; c.o_up = P.o_up; c.o_cf = P.o_cf;
  double* g = wsd + (size_t)blockIdx.x * P.g_doubles;
  c.qd = g + P.g_qd; c.ps = g + P.g_ps; c.x = g + P.g_x; c.dx = g + P.g_dx; c.rx = g + P.g_rx;
  c.y = g + P.g_y; c.dy = g + P.g_dy; c.ry = g + P.g_ry; c.cg = g + P.g_cg;
  c.z = g + P.g_z; c.s = g + P.g_s; c.d = g + P.g_d; c.rz = g + P.g_rz; c.rs = g + P.g_rs; c.dz = g + P.g_dz;
  c.ds = g + P.g_ds; c.t = g + P.g_t; c.h = g + P.g_h; c.W = g + P.g_W; c.E = g + P.g_E;
  c.Kb = g + P.g_Kb; c.KbT = g + P.g_KbT; c.Brow = g + P.g_Brow; c.Bcol = g + P.g_Bcol; c.Cn = g + P.g_Cn; c.FB = g + P.g_FB;
  int* gi = wsi + (size_t)blockIdx.x * P.i_ints;
  c.deg = gi + P.i_deg; c.start = gi + P.i_start; c.adj = gi + P.i_adj;
  c.nb = P.nb; c.n = P.n; c.e = P.e; c.cs = P.cs; c.ncap = P.ncap;
}

__global__ void __launch_bounds__(NT, 1) band_forward_kernel(const __grid_constant__ BArgs a) {
  const BPlan& P = a.P;
  Ctx c;
  init_ctx(c, P, a.wsd, a.wsi);
  BProf pf;
  pf.start(a.prof ? a.prof + (size_t)blockIdx.x * BPH_COUNT : nullptr);
  for (int sc = blockIdx.x; sc < a.B; sc += gridDim.x) {
    const int ncs = a.soa.nc;
    c.nc = a.soa.nc_s ? a.soa.nc_s[sc] : ncs;
    c.b1 = a.soa.b1 + (a.soa.nc_s ? (size_t)sc * ncs : 0);
    c.b2 = a.soa.b2 + (a.soa.nc_s ? (size_t)sc * ncs : 0);
    c.A = P.e > 0 ? a.A + (size_t)sc * P.e * P.n : nullptr;
    int rc = (c.nc < 0 || c.nc > P.ncap) ? 1 : 0;
    if (rc == 0) { c.m = c.cs * c.nc; rc = build_structure(c, a.soa, sc); }
    pf.lap(BPH_STRUCT);
    if (pf.dst && threadIdx.x == 0 && rc == 0) atomicAdd((unsigned long long*)&pf.dst[BPH_GRADS], (unsigned long long)c.bw);   // (debug: half bandwidth)
    if (rc != 0) {
      if (threadIdx.x == 0) { a.status[sc] = rc == 2 ? -1 : STATUS_UNSUPPORTED; a.iters[sc] = 0; if (a.resid) a.resid[sc] = nan(""); }
    } else {
      forward_scene(a, c, pf, sc);
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------ backward (lcp.py:37-64), one scene
// One factorisation at d = lam / slack (clamped to [1e-10, 1e10] like the condensed fp64 backward, DESIGN.md
// section 3.1), one solve with the right-hand side (dl/dzhat, 0, 0, 0), then the chain rule through the assembly
// (world.py:144-234, engines.py:50-116) applied to the factored gradients of lcp.py:52-63 -- evaluated only at
// the entries the assembly writes (same formulas as lcp_condensed.cuh's engine path). flags bit 0 (exact adjoint)
// factors and solves the transposed system K^T instead (DESIGN.md section 3.4); the chain rule is the same.
//
// Zero gradients of the contact slot at output offset oc (an unused slot, or a scene the forward rejected).
__device__ __forceinline__ void zero_contact_grads(const BBwdArgs& a, size_t oc) {
  if (a.dnormal) { a.dnormal[oc * 2] = 0; a.dnormal[oc * 2 + 1] = 0; }
  if (a.dp1) { a.dp1[oc * 2] = 0; a.dp1[oc * 2 + 1] = 0; }
  if (a.dp2) { a.dp2[oc * 2] = 0; a.dp2[oc * 2 + 1] = 0; }
  if (a.drest) a.drest[oc] = 0;
  if (a.dmu) a.dmu[oc] = 0;
}

// The gradients of one cotangent from the solve's dx, dlam, dnu in c: inputs of scene sc, outputs at row so.
__device__ __forceinline__ void backward_grads(const BBwdArgs& a, Ctx& c, BProf& pf, int sc, int so) {
  const int tid = threadIdx.x, n = c.n, e = c.e, nc = c.nc, ncap = c.ncap, nb = c.nb;
  const cnd::EngineSoA<double>& E = a.soa;
  const int ncs = E.nc, mode = E.mode;
  const double* zh = a.zhat + (size_t)sc * n;
  const double* dx = c.dx;
  const double* dlam = c.dz;
  const double* lm = c.z;
  const double* v = E.v + (size_t)sc * n;
  for (int k = tid; k < ncs; k += NT) {
    const size_t ic = (size_t)sc * ncs + k, oc = (size_t)so * ncs + k;
    if (k >= nc) {                                                          // unused slots of a scene with fewer contacts
      zero_contact_grads(a, oc);
      continue;
    }
    const double nx = E.normal[ic * 2], ny = E.normal[ic * 2 + 1];
    const double p1x = E.p1[ic * 2], p1y = E.p1[ic * 2 + 1], p2x = E.p2[ic * 2], p2y = E.p2[ic * 2 + 1];
    const bool two = c.b2[k] < nb;                                          // else body2 is a static obstacle: no dofs
    const int j1 = 3 * c.b1[k], j2 = two ? 3 * c.b2[k] : j1;
    const double rc = E.rest[ic];
    const double dhc = -dlam[k];                                            // dh = -dlam  (:55)
    double gnx = 0, gny = 0, g1x = 0, g1y = 0, g2x = 0, g2y = 0, jcv = 0;
    const int nrows = mode == 0 ? 3 : 1;
    for (int q = 0; q < nrows; ++q) {
      const double ddx_ = q == 0 ? nx : (q == 1 ? ny : -ny), ddy_ = q == 0 ? ny : (q == 1 ? -nx : nx);
      const double dl = dlam[q * ncap + k], lq = lm[q * ncap + k];
      double g[6];
#pragma unroll
      for (int t = 0; t < 3; ++t) {
        g[t] = dl * zh[j1 + t] + lq * dx[j1 + t];                           // dG[i][j1 + t]  (:53)
        g[3 + t] = two ? dl * zh[j2 + t] + lq * dx[j2 + t] : 0.0;
      }
      if (q == 0) {
        const double row[6] = {p1x * ddy_ - p1y * ddx_, ddx_, ddy_, -(p2x * ddy_ - p2y * ddx_), -ddx_, -ddy_};
#pragma unroll
        for (int t = 0; t < 3; ++t) jcv += row[t] * v[j1 + t] + row[3 + t] * (two ? v[j2 + t] : 0.0);
        const double hs_ = mode == 0 ? rc : (1.0 - rc);                     // h_c = (Jc v) rest  |  (Jc v)(1 - rest)
#pragma unroll
        for (int t = 0; t < 3; ++t) { g[t] += dhc * hs_ * v[j1 + t]; g[3 + t] += dhc * hs_ * (two ? v[j2 + t] : 0.0); }
      }
      const double gdx = -p1y * g[0] + g[1] + p2y * g[3] - g[4];
      const double gdy = p1x * g[0] + g[2] - p2x * g[3] - g[5];
      g1x += ddy_ * g[0]; g1y += -ddx_ * g[0];
      g2x += -ddy_ * g[3]; g2y += ddx_ * g[3];
      if (q == 0) { gnx += gdx; gny += gdy; }
      else if (q == 1) { gny += gdx; gnx += -gdy; }                         // dir1 = (ny, -nx)
      else { gny += -gdx; gnx += gdy; }                                     // dir2 = (-ny, nx)
    }
    if (a.dnormal) { a.dnormal[oc * 2] = gnx; a.dnormal[oc * 2 + 1] = gny; }
    if (a.dp1) { a.dp1[oc * 2] = g1x; a.dp1[oc * 2 + 1] = g1y; }
    if (a.dp2) { a.dp2[oc * 2] = g2x; a.dp2[oc * 2 + 1] = g2y; }
    if (a.drest) a.drest[oc] = mode == 0 ? dhc * jcv : -dhc * jcv;
    if (a.dmu) a.dmu[oc] = mode == 0 ? -(dlam[3 * ncap + k] * lm[k]) : 0.0;   // dF[gamma_c][c]  (:54)
  }
  for (int body = tid; body < nb; body += NT) {
    double dm = 0.0;
    const int s0 = c.start[body], s1 = c.start[body + 1];
#pragma unroll
    for (int comp = 0; comp < 3; ++comp) {
      const int j = 3 * body + comp;
      const double md = comp == 0 ? E.inertia[(size_t)sc * nb + body] : E.mass[(size_t)sc * nb + body];
      const double dpj = mode == 0 ? dx[j] : 0.0;                           // dp = dx (:52); post-stabilisation has p = 0
      if (a.dfext) a.dfext[(size_t)so * n + j] = E.dt * dpj;
      if (a.dv) {
        double acc = md * dpj;
        for (int it = s0; it < s1; ++it) {                                  // the contacts that touch this body
          const int ad = c.adj[it], k = ad >> 1, side = ad & 1;
          const double hs_ = mode == 0 ? E.rest[(size_t)sc * ncs + k] : (1.0 - E.rest[(size_t)sc * ncs + k]);
          acc += -dlam[k] * hs_ * c.cg[12 * (size_t)k + 3 * side + comp];  // dh_c d(h_c)/dv_j
        }
        a.dv[(size_t)so * n + j] = acc;
      }
      const double dq = dx[j] * zh[j] + dpj * v[j];                         // dQ_jj = 1/2 (dx_j z_j + z_j dx_j)  (:61), dp_j d(p_j)/dM_jj
      if (comp == 0) { if (a.dinertia) a.dinertia[(size_t)so * nb + body] = dq; }
      else dm += dq;
    }
    if (a.dmass) a.dmass[(size_t)so * nb + body] = dm;
  }
  if (a.db && e > 0) for (int i = tid; i < e; i += NT) a.db[(size_t)so * e + i] = -c.dy[i];
  if (a.dA && e > 0) {
    double* o = a.dA + (size_t)so * e * n;
    for (int i = 0; i < e; ++i)
      for (int j = tid; j < n; j += NT) o[(size_t)i * n + j] = c.dy[i] * zh[j] + c.y[i] * dx[j];
  }
  __syncthreads();
  pf.lap(BPH_GRADS);
}

// The saved solution of scene sc (zhat, lam, slack, nu of BBwdArgs or BJvpArgs) into c.x, c.z, c.s, c.y -- the
// rows of contact k move from out_row to slot-major r ncap + k -- with d = lam / slack clamped to [1e-10, 1e10] as in
// the condensed fp64 backward and c.rs zeroed, then one factorisation of K (trans: K^T, the exact adjoint).
template <typename Args>
__device__ __forceinline__ void factor_saved(const Args& a, Ctx& c, BProf& pf, int sc, bool trans) {
  const int tid = threadIdx.x, n = c.n, e = c.e, nc = c.nc, cs = c.cs, ncap = c.ncap;
  const cnd::EngineSoA<double>& E = a.soa;
  const double* mu = E.mu ? E.mu + (size_t)sc * E.nc : nullptr;
  const double* zh = a.zhat + (size_t)sc * n;
  const double* lamv = a.lam + (size_t)sc * a.P.m;
  const double* slk = a.slack + (size_t)sc * a.P.m;
  for (int i = tid; i < n; i += NT) c.x[i] = zh[i];
  for (int r = 0; r < cs; ++r)
    for (int k = tid; k < nc; k += NT) {
      const int i = r * ncap + k, o = out_row(r, k, nc);
      double d = lamv[o] / slk[o];                                          // :44
      d = d > 1e10 ? 1e10 : (d < 1e-10 ? 1e-10 : d);
      c.z[i] = lamv[o]; c.s[i] = slk[o]; c.d[i] = d; c.rs[i] = 0.0;
    }
  for (int i = tid; i < e; i += NT) c.y[i] = a.nu[(size_t)sc * e + i];
  __syncthreads();
  factor_kkt(c, pf, E.mode, mu, trans);                                     // :46
}

// Binds scene sc's contacts to c and finds its structure: 0 = ok, 1 = unsupported (too many contacts or the
// topology), 2 = singular mass matrix.
__device__ __forceinline__ int bind_scene(Ctx& c, const BPlan& P, const cnd::EngineSoA<double>& soa, const double* A,
                                          int sc) {
  const int ncs = soa.nc;
  c.nc = soa.nc_s ? soa.nc_s[sc] : ncs;
  c.b1 = soa.b1 + (soa.nc_s ? (size_t)sc * ncs : 0);
  c.b2 = soa.b2 + (soa.nc_s ? (size_t)sc * ncs : 0);
  c.A = P.e > 0 ? A + (size_t)sc * P.e * P.n : nullptr;
  int rc = (c.nc < 0 || c.nc > P.ncap) ? 1 : 0;
  if (rc == 0) { c.m = c.cs * c.nc; rc = build_structure(c, soa, sc); }
  return rc;
}

// One factorisation at the saved solution, then one solve and chain rule per cotangent r in [r0, r1); each
// round streams the factor blocks back from the L2 workspace.
__device__ __forceinline__ void backward_scene(const BBwdArgs& a, Ctx& c, BProf& pf, int sc, int r0, int r1) {
  const int tid = threadIdx.x, n = c.n;
  factor_saved(a, c, pf, sc, (a.flags & 1u) != 0);
  for (int r = r0; r < r1; ++r) {
    const int so = r * a.B + sc;
    for (int i = tid; i < n; i += NT) c.rx[i] = a.g[(size_t)so * n + i];
    __syncthreads();
    solve_kkt(c, pf, c.rx, c.rs, nullptr, nullptr, c.dx, c.ds, c.dz, c.dy);   // :47-50 (c.W holds W^T when exact)
    backward_grads(a, c, pf, sc, so);
  }
}

__global__ void __launch_bounds__(NT, 1) band_backward_kernel(const __grid_constant__ BBwdArgs a) {
  const BPlan& P = a.P;
  Ctx c;
  init_ctx(c, P, a.wsd, a.wsi);
  BProf pf;
  pf.start(a.prof ? a.prof + (size_t)blockIdx.x * BPH_COUNT : nullptr);
  for (int w = blockIdx.x; w < a.B * a.chunks; w += gridDim.x) {
    const int sc = w / a.chunks, ch = w - sc * a.chunks;
    const int r0 = (int)((long long)a.R * ch / a.chunks), r1 = (int)((long long)a.R * (ch + 1) / a.chunks);
    const int ncs = a.soa.nc, n = P.n, nb = P.nb, e = P.e;
    const int rc = bind_scene(c, P, a.soa, a.A, sc);
    pf.lap(BPH_STRUCT);
    if (rc != 0) {                                                          // the forward reported it: zero gradients
      const int tid = threadIdx.x;
      for (int r = r0; r < r1; ++r) {
        const size_t so = (size_t)r * a.B + sc;
        for (int i = tid; i < n; i += NT) { if (a.dv) a.dv[so * n + i] = 0; if (a.dfext) a.dfext[so * n + i] = 0; }
        for (int i = tid; i < nb; i += NT) { if (a.dmass) a.dmass[so * nb + i] = 0; if (a.dinertia) a.dinertia[so * nb + i] = 0; }
        for (int i = tid; i < ncs; i += NT) zero_contact_grads(a, so * ncs + i);
        for (int i = tid; i < e; i += NT) if (a.db) a.db[so * e + i] = 0;
        if (a.dA) for (int i = tid; i < e * n; i += NT) a.dA[so * e * n + i] = 0;
      }
    } else {
      backward_scene(a, c, pf, sc, r0, r1);
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------ Jacobian-vector products (DESIGN.md section 8)
// Same system as lcp_condensed.cuh's cond_jvp_kernel: K [dx; ds; dz; dy] = -(r_x, 0, r_z, r_y) with the
// non-transposed K factored once per (scene, chunk of tangents) at the saved iterate, d clamped as in the backward.
// The right-hand side is cnd::engine_jvp_rhs with this layout: rows slot-major (row q of contact k at q ncap + k),
// and the contacts of a dof are those of its body's adjacency.
struct BandRows {
  const Ctx& c;
  __device__ __forceinline__ double* x() const { return c.x; }
  __device__ __forceinline__ double* z() const { return c.z; }
  __device__ __forceinline__ double* y() const { return c.y; }
  __device__ __forceinline__ double* rx() const { return c.rx; }
  __device__ __forceinline__ double* rz() const { return c.rz; }
  __device__ __forceinline__ double* ry() const { return c.ry; }
  __device__ __forceinline__ int row(int q, int k) const { return q * c.ncap + k; }
  template <typename F>
  __device__ __forceinline__ void walk(int, int body, F f) const {
    const int s0 = c.start[body], s1 = c.start[body + 1];
    for (int it = s0; it < s1; ++it) { const int ad = c.adj[it]; f(ad >> 1, ad & 1); }
  }
};

// engine_jvp_rhs in the banded layout, kept out of line as in the condensed kernel.
__device__ __noinline__ void jvp_rhs(const BJvpArgs& a, const Ctx& c, int sc, int so) {
  cnd::engine_jvp_rhs<double>(a.soa, a.t, BandRows{c}, sc, so, c.n, c.e, c.nc);
}

// The saved solution and one factorisation of K, then one right-hand side and one solve per tangent r in [r0, r1).
__device__ __forceinline__ void jvp_scene(const BJvpArgs& a, Ctx& c, BProf& pf, int sc, int r0, int r1) {
  const int tid = threadIdx.x, n = c.n, e = c.e;
  factor_saved(a, c, pf, sc, false);
  for (int r = r0; r < r1; ++r) {
    const size_t so = (size_t)r * a.B + sc;
    jvp_rhs(a, c, sc, (int)so);
    solve_kkt(c, pf, c.rx, c.rs, c.rz, e > 0 ? c.ry : nullptr, c.dx, c.ds, c.dz, c.dy);
    for (int i = tid; i < n; i += NT) a.dz[so * n + i] = c.dx[i];
    __syncthreads();
    pf.lap(BPH_GRADS);
  }
}

__global__ void __launch_bounds__(NT, 1) band_jvp_kernel(const __grid_constant__ BJvpArgs a) {
  const BPlan& P = a.P;
  Ctx c;
  init_ctx(c, P, a.wsd, a.wsi);
  BProf pf;
  pf.start(a.prof ? a.prof + (size_t)blockIdx.x * BPH_COUNT : nullptr);
  for (int w = blockIdx.x; w < a.B * a.chunks; w += gridDim.x) {
    const int sc = w / a.chunks, ch = w - sc * a.chunks;
    const int r0 = (int)((long long)a.R * ch / a.chunks), r1 = (int)((long long)a.R * (ch + 1) / a.chunks);
    const int rc = bind_scene(c, P, a.soa, a.A, sc);
    pf.lap(BPH_STRUCT);
    if (rc != 0) {                                                          // the forward reported it: zero tangents
      for (int r = r0; r < r1; ++r)
        for (int i = threadIdx.x; i < P.n; i += NT) a.dz[((size_t)r * a.B + sc) * P.n + i] = 0.0;
    } else {
      jvp_scene(a, c, pf, sc, r0, r1);
    }
    __syncthreads();
  }
}

#endif  // LCP_BAND_DEVICE

}  // namespace bnd
}  // namespace lcpb200
