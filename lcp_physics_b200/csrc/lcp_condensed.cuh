// lcp_condensed.cuh -- "condensed KKT" PDIPM kernels: the structured fast path of the solver.
//
// Same algorithm as lcp_solver.cuh (pdipm.py:49-186, :325-454; lcp.py:22-64) but the Newton system
// of every iteration is reduced to the PRIMAL side instead of the dual side. The reference
// eliminates dx and factors the m x m matrix T = G Q^-1 G^T + F + diag(s/z) (pdipm.py:414-454); every
// LCP the engine builds (engines.py:50-76, :80-116) has two properties this file exploits:
//   (1) F + diag(s/z) =: M is block diagonal after a row permutation -- the connected components
//       of F's sparsity graph are the per-contact blocks {normal, friction dirs, gamma}
//       (engines.py:66-72: E, mu, -E^T), size 2 + fd; for post-stabilisation F = 0 (size 1);
//   (2) a component's rows of G touch two bodies only (world.py:172-211): <= 6 columns (3 for a one-body contact
//       against a static obstacle, body2 >= nb).
// Eliminating dz = M^-1 (G dx + rz - rs/d) instead gives the n x n (+ e equality rows) system
//       [ Q + G^T M^-1 G   A^T ] [dx]   [ -rx - G^T M^-1 (rz - rs/d) ]
//       [ A                0   ] [dy] = [ -ry                        ]
// n = 96 instead of m = 256 at BASELINE config 3: 19x fewer factorisation flops, and the matrix is
// small enough for two scenes per SM. The same linear system is solved, so the iterates are the
// reference's up to round-off. Round-off is the catch: M^-1 has entries z/s up to 1e13 (fp32 runs)
// on active constraints and K = Q + G^T M^-1 G inherits them, so K is formed, factored and solved
// in FP64 whatever the I/O dtype (H100: FP64 FMA at half the FP32 rate). Measured on seeded
// config-3 scenes (DESIGN.md "Parity"): fp32 I/O + fp64 K is CLOSER to the fp64 reference than the
// reference's own fp32 run; an fp32 K is 20x worse than it; explicit inverses of 16x16 (even 4x4)
// diagonal blocks of the factors lose 4-6 digits, so the triangular solves are exact
// substitutions.
//
// Scenes whose inputs do not have this structure (dense F or G, non-diagonal Q, n + e > 128) are
// flagged and solved by the dual-form kernels of lcp_solver.cuh (the structure test is per scene,
// on the device, on the dense tensors the API receives).
//
// Execution: one CTA of 256 threads per scene, persistent grid, two CTAs per SM at n + e <= 96.
//   * structure (once per scene): ballot scans compact F and G rows, label propagation finds F's
//     components, rows are regrouped per component: Gd (dense cs x <= 8 block + its column list),
//     Fd (cs x cs), per-column lists of (component, slot) for G^T w and the assembly of K;
//   * per iteration: W_c = (Fd_c + diag(s/z))^-1 per component (fp64, Gauss-Jordan with partial
//     pivoting in registers), K assembled in shared memory (column major), moved to REGISTERS in a
//     2-D cyclic layout (thread (ti,tj) owns K[16r+ti][16c+tj]), LU without pivoting, two pivots
//     per CTA barrier (pivot rows/columns broadcast through shared memory, every thread redoes the
//     2x2 pivot arithmetic), factors written back transposed with U's columns pre-scaled by 1/u_kk;
//   * solves: ONE warp, exact forward/back substitution, 4 pivots per shuffle round (the 4x4
//     diagonal piece is redone by every lane, so the dependent chain per pivot is ~14 cycles).
#pragma once
#include "lcp_device.cuh"

namespace lcpb200 {
namespace cnd {

constexpr int NT = 256;          // threads per CTA (16 x 16 grid over K)
constexpr int UC = 8;            // max distinct columns of G over the rows of one component
constexpr int CSMAX = 6;         // max rows per component of F
constexpr int KS = 8;            // scan slots per row of F / G
constexpr int LMAX = 16;         // max (component, slot) entries per column of G
constexpr int LU_BW = 2;         // block band (16 x 16 blocks) of the band LU, factor_K_body<NS, LU_BW>
constexpr int MISC_BAND_LU = 4;  // S.misc() slot set by mark_band_lu: 1 = factor this scene's K with the band LU
constexpr int CFLAG_DENSE_LU = 4;          // CPlan::flags bit: dense LU for every scene (the reference the tests compare the band LU against)
constexpr int STATUS_UNSUPPORTED = -100;   // internal: scene left to the dual-form kernel

// ------------------------------------------------------------------ launch plan / shared layout
struct CPlan {
  int ok;                     // 0: the condensed path is not available for this (dtype, n, m, e)
  int n, m, e, N, NP, NS;
  int pcap;                   // capacity of component-sorted row positions
  int wcap;                   // capacity (elements) of W and Fd
  int smem_bytes;
  int ctas_per_sm;
  int flags;                  // experiment switches (LCPB200_COND_FLAGS): 1 = 1/d in fp64, 2 = rz - rs/d in fp64,
                              // 4 = dense LU for every scene (CFLAG_DENSE_LU)
  int sbytes;                 // bytes of one scene's saved structure (save_structure / load_structure)
  // byte offsets into the dynamic shared memory (filled by carve_plan)
  int o_K, o_W, o_scr, o_bx, o_rdiag, o_Fd, o_Gd, o_As, o_x, o_rx, o_dx, o_qd, o_y, o_ry, o_dy,
      o_s, o_z, o_d, o_rz, o_ds, o_dz, o_rs2, o_red, o_rows, o_posof, o_clist, o_ccols, o_ncols, o_clcnt, o_misc;
};

__host__ __device__ inline size_t al16(size_t x) { return (x + 15) & ~(size_t)15; }
// structure-build scratch: Fi,Gi (u16 KS*m each), Fv,Gv (T KS*m each), 5 int arrays of m, member
// lists (u16 CSMAX*m), column bitmaps (8 words per component), unsorted column lists (u16 LMAX*n + n ints)
__host__ __device__ inline size_t scratch_bytes(int n, int m, int tsize) {
  return al16((size_t)2 * KS * m * 2) + al16((size_t)2 * KS * m * tsize) + al16((size_t)5 * m * 4) +
         al16((size_t)CSMAX * m * 2) + al16((size_t)8 * m * 4) + al16((size_t)LMAX * n * 2) + al16((size_t)n * 4) + 64;
}

// Lays the shared memory out (offsets into P) and returns the total. tsize = sizeof(T).
inline size_t carve_plan(CPlan& P, int tsize) {
  size_t o = 0;
  const int n = P.n, m = P.m, e = P.e, NP = P.NP, pcap = P.pcap, wcap = P.wcap;
#define CND_TAKE(field, bytes) do { P.field = (int)o; o += al16((size_t)(bytes)); } while (0)
  size_t kb = (size_t)NP * NP * 8;                              // K | structure scratch | LU broadcast buffers
  if (scratch_bytes(n, m, tsize) > kb) kb = scratch_bytes(n, m, tsize);
  if ((size_t)8 * NP * 8 > kb) kb = (size_t)8 * NP * 8;
  { const size_t qn = (NP + 31) / 32, sl = (size_t)(NP / qn) * qn * qn * 32 * 8; if (sl > kb) kb = sl; }   // SolveLayout
  CND_TAKE(o_K, kb);
  CND_TAKE(o_W, (size_t)wcap * 8);
  CND_TAKE(o_scr, (size_t)pcap * 8);
  CND_TAKE(o_bx, (size_t)NP * 8);
  CND_TAKE(o_rdiag, (size_t)NP * 8);
  CND_TAKE(o_Fd, (size_t)wcap * tsize);
  CND_TAKE(o_Gd, (size_t)UC * pcap * tsize);
  CND_TAKE(o_As, (size_t)e * n * tsize);
  CND_TAKE(o_x, n * tsize); CND_TAKE(o_rx, n * tsize); CND_TAKE(o_dx, n * tsize); CND_TAKE(o_qd, n * tsize);
  CND_TAKE(o_y, e * tsize); CND_TAKE(o_ry, e * tsize); CND_TAKE(o_dy, e * tsize);
  CND_TAKE(o_s, m * tsize); CND_TAKE(o_z, m * tsize); CND_TAKE(o_d, m * tsize); CND_TAKE(o_rz, m * tsize);
  CND_TAKE(o_ds, m * tsize); CND_TAKE(o_dz, m * tsize); CND_TAKE(o_rs2, m * tsize);
  CND_TAKE(o_red, 192 * tsize);
  CND_TAKE(o_rows, pcap * 2);
  CND_TAKE(o_posof, m * 2);
  CND_TAKE(o_clist, LMAX * n * 2);
  CND_TAKE(o_ccols, UC * pcap);
  CND_TAKE(o_ncols, pcap);
  CND_TAKE(o_clcnt, n);
  CND_TAKE(o_misc, 16 * 4);
#undef CND_TAKE
  // what build_structure leaves behind: {Struct} + [Fd, Gd, As] + [qd] + [rows, posof, clist, ccols, ncols, clcnt]
  P.sbytes = 16 + (P.o_x - P.o_Fd) + (P.o_y - P.o_qd) + (P.o_misc - P.o_rows);
  return o;
}

extern __shared__ __align__(16) unsigned char cnd_smem[];

// Accessors: every array is cnd_smem + an offset that lives in the kernel parameters (constant
// bank), so no pointer is kept in a register across phases.
template <typename T>
struct CSmem {
  const CPlan& P;
  __device__ __forceinline__ explicit CSmem(const CPlan& p) : P(p) {}
#define CND_ACC(name, type) __device__ __forceinline__ type* name() const { return reinterpret_cast<type*>(cnd_smem + P.o_##name); }
  CND_ACC(K, double) CND_ACC(W, double) CND_ACC(scr, double) CND_ACC(bx, double) CND_ACC(rdiag, double)
  CND_ACC(Fd, T) CND_ACC(Gd, T) CND_ACC(As, T)
  CND_ACC(x, T) CND_ACC(rx, T) CND_ACC(dx, T) CND_ACC(qd, T) CND_ACC(y, T) CND_ACC(ry, T) CND_ACC(dy, T)
  CND_ACC(s, T) CND_ACC(z, T) CND_ACC(d, T) CND_ACC(rz, T) CND_ACC(ds, T) CND_ACC(dz, T) CND_ACC(rs2, T)
  CND_ACC(red, T)
  CND_ACC(rows, unsigned short) CND_ACC(posof, unsigned short) CND_ACC(clist, unsigned short)
  CND_ACC(ccols, unsigned char) CND_ACC(ncols, unsigned char) CND_ACC(clcnt, unsigned char)
  CND_ACC(misc, int)
#undef CND_ACC
};

// per-scene structure facts (uniform across the CTA, kept in registers)
struct Struct {
  int ncomp, cs;              // components, rows per component (uniform stride; short ones padded)
  int sh;                     // log2 of the smallest power of two >= ncomp: (r, c) = (t >> sh, t & mask) without divisions
  int m;                      // inequality rows of THIS scene (== P.m, or 4 nc_s / nc_s on the engine path with per-scene contact counts)
};

// optional per-phase SM cycle counters (thread 0 of every CTA; lcpb200_profile). A compile-time switch: the
// kernels are instantiated twice, and the production instantiation carries no profiling state (a pointer and a
// timestamp live across every phase cost registers the LU and the solves need).
// The last two slots are counts, not cycles: the factorisations and the solves (forward + backward substitution)
// the forward kernel executed.
enum { CPH_STRUCT = 0, CPH_WINV, CPH_ASSEMBLE, CPH_LU, CPH_SOLVE_RHS, CPH_SOLVE_TRI, CPH_SOLVE_POST, CPH_RESID,
       CPH_STEP, CPH_GRADS, CPH_FACTORS, CPH_SOLVES, CPH_COUNT };
template <bool ON>
struct Prof {
  long long* p;               // this CTA's CPH_COUNT counters
  long long t;
  __device__ __forceinline__ explicit Prof(long long* p_) : p(p_), t(0) {}
  __device__ __forceinline__ void start() { if (threadIdx.x == 0) t = clock64(); }
  __device__ __forceinline__ void lap(int ph) {
    if (threadIdx.x == 0) {
      const long long n = clock64();
      atomicAdd(reinterpret_cast<unsigned long long*>(p + ph), (unsigned long long)(n - t));   // no dependent load
      t = n;
    }
  }
  __device__ __forceinline__ void count(int ph, int k = 1) {
    if (threadIdx.x == 0) atomicAdd(reinterpret_cast<unsigned long long*>(p + ph), (unsigned long long)k);
  }
};
template <>
struct Prof<false> {
  __device__ __forceinline__ explicit Prof(long long*) {}
  __device__ __forceinline__ void start() {}
  __device__ __forceinline__ void lap(int) {}
  __device__ __forceinline__ void count(int, int = 1) {}
};

// ------------------------------------------------------------------ structure detection
// Scans one dense row-major matrix (rows x cols) into KS-slot row lists (values + column indices),
// one warp per row, RP rows (all their loads) in flight per warp; ordered, hence deterministic.
// Returns non-zero if a row has > KS entries.
template <typename T>
__device__ __forceinline__ int scan_rows(const T* __restrict__ A, int rows, int cols, T* vals, unsigned short* idx,
                                         int* cnt) {
  constexpr int CH = 8, RP = (sizeof(T) == 8) ? 2 : 4;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = NT >> 5;
  int bad = 0;
  if (cols <= 32 * CH) {
    for (int r0 = warp * RP; r0 < rows; r0 += nw * RP) {
      T v[RP][CH];
#pragma unroll
      for (int rr = 0; rr < RP; ++rr) {
        const T* row = A + (size_t)min(r0 + rr, rows - 1) * cols;
#pragma unroll
        for (int q = 0; q < CH; ++q) { const int j = q * 32 + lane; v[rr][q] = j < cols ? row[j] : T(0); }
      }
#pragma unroll
      for (int rr = 0; rr < RP; ++rr) {
        const int r = r0 + rr;
        if (r >= rows) break;
        int c = 0;
#pragma unroll
        for (int q = 0; q < CH; ++q) {
          const bool nz = v[rr][q] != T(0);
          const unsigned mask = __ballot_sync(FULL, nz);
          const int pos = c + __popc(mask & ((1u << lane) - 1u));
          if (nz && pos < KS) { vals[pos * rows + r] = v[rr][q]; idx[pos * rows + r] = (unsigned short)(q * 32 + lane); }
          c += __popc(mask);
        }
        if (c > KS) bad = 1;
        if (lane == 0) cnt[r] = c;
      }
    }
    return bad;
  }
  for (int r = warp; r < rows; r += nw) {
    const T* row = A + (size_t)r * cols;
    int c = 0;
    for (int j0 = 0; j0 < cols; j0 += 32 * CH) {
      T v[CH];
#pragma unroll
      for (int q = 0; q < CH; ++q) { const int j = j0 + q * 32 + lane; v[q] = j < cols ? row[j] : T(0); }
#pragma unroll
      for (int q = 0; q < CH; ++q) {
        const bool nz = v[q] != T(0);
        const unsigned mask = __ballot_sync(FULL, nz);
        const int pos = c + __popc(mask & ((1u << lane) - 1u));
        if (nz && pos < KS) { vals[pos * rows + r] = v[q]; idx[pos * rows + r] = (unsigned short)(j0 + q * 32 + lane); }
        c += __popc(mask);
      }
    }
    if (c > KS) bad = 1;
    if (lane == 0) cnt[r] = c;
  }
  return bad;
}

__device__ __forceinline__ void prefetch_l2(const void* p, size_t bytes) {
  const char* c = reinterpret_cast<const char*>(p);
  for (size_t o = (size_t)threadIdx.x * 128; o < bytes; o += (size_t)NT * 128)
    asm volatile("prefetch.global.L2 [%0];" ::"l"(c + o));
}

// Builds the per-scene structure in shared memory. Returns false (uniformly) when the scene does
// not have the structure this path needs. *singular is set when Q has a zero / non-finite diagonal
// entry (the reference fails its LU of Q, pdipm.py:361-368).
template <typename T>
__device__ __noinline__ bool build_structure(const CPlan& P, CSmem<T>& S, Struct& st, const T* __restrict__ Q,
                                             const T* __restrict__ G, const T* __restrict__ A,
                                             const T* __restrict__ F, int* singular) {
  const int n = P.n, m = P.m, e = P.e, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, pcap = P.pcap;
  // the inputs are read exactly once, here: pull them towards L2 before the first dependent load
  prefetch_l2(F, (size_t)m * m * sizeof(T));
  prefetch_l2(G, (size_t)m * n * sizeof(T));
  prefetch_l2(Q, (size_t)n * n * sizeof(T));
  // scratch carved from the K region
  char* sb = reinterpret_cast<char*>(S.K());
  unsigned short* Fi = reinterpret_cast<unsigned short*>(sb);
  unsigned short* Gi = Fi + (size_t)KS * m;
  size_t o = al16((size_t)2 * KS * m * 2);
  T* Fv = reinterpret_cast<T*>(sb + o);
  T* Gv = Fv + (size_t)KS * m;
  o += al16((size_t)2 * KS * m * sizeof(T));
  int* Fcnt = reinterpret_cast<int*>(sb + o);
  int* Gcnt = Fcnt + m;
  int* label = Gcnt + m;
  int* cidx = label + m;       // component index of a root row
  int* memcnt = cidx + m;      // rows of the component rooted at row l
  o += al16((size_t)5 * m * 4);
  unsigned short* memb = reinterpret_cast<unsigned short*>(sb + o);      // [m][CSMAX] member rows, unordered
  o += al16((size_t)CSMAX * m * 2);
  unsigned* cmap = reinterpret_cast<unsigned*>(sb + o);                  // [ncomp][8] column bitmaps
  o += al16((size_t)8 * m * 4);
  unsigned short* cl_tmp = reinterpret_cast<unsigned short*>(sb + o);    // [LMAX][n] unsorted column lists
  o += al16((size_t)LMAX * n * 2);
  int* cl_cnt = reinterpret_cast<int*>(sb + o);
  int* flags = S.misc();       // [0..7] flags, [8..15] warp totals

  if (tid < 16) flags[tid] = 0;
  // ---- Q must be diagonal (every mass matrix world.py:57-61 builds)
  int bad = 0;
  for (int t = tid; t < n * n; t += NT) {
    const int i = t / n, j = t - i * n;
    const T q = Q[t];
    if (i == j) {
      S.qd()[i] = q;
      if (!(q != T(0) && isfinite((double)q))) bad |= 2;
    } else if (q != T(0)) bad |= 1;
  }
  bad |= scan_rows<T>(F, m, m, Fv, Fi, Fcnt) ? 1 : 0;
  bad |= scan_rows<T>(G, m, n, Gv, Gi, Gcnt) ? 1 : 0;
  for (int t = tid; t < e * n; t += NT) S.As()[t] = A[t];
  for (int i = tid; i < m; i += NT) { label[i] = i; memcnt[i] = 0; }
  for (int a = tid; a < n; a += NT) cl_cnt[a] = 0;
  const int anybad = __syncthreads_or(bad);
  if (anybad & 2) { *singular = 1; return false; }
  if (anybad & 1) return false;

  // ---- components of F's sparsity graph: label propagation to the minimum row index
  for (int pass = 0; pass < 64; ++pass) {
    int changed = 0;
    for (int i = tid; i < m; i += NT) {
      const int c = Fcnt[i];
      int li = ((volatile int*)label)[i];
      for (int k = 0; k < c; ++k) {
        const int j = Fi[k * m + i];
        const int lj = ((volatile int*)label)[j];
        if (lj < li) { li = lj; changed = 1; }
        else if (li < lj) { atomicMin(&label[j], li); changed = 1; }
      }
      atomicMin(&label[i], li);
    }
    if (!__syncthreads_or(changed)) break;
    if (pass == 63) return false;
  }
  // ---- component index = rank of the root among roots (ballot prefix sums); member lists
  if (m > 4 * NT) return false;
  int running = 0;
  for (int base = 0; base < m; base += NT) {
    const int i = base + tid;
    const bool root = i < m && label[i] == i;
    const unsigned mask = __ballot_sync(FULL, root);
    if (lane == 0) flags[8 + warp] = __popc(mask);
    __syncthreads();
    int before = running;
    for (int w = 0; w < warp; ++w) before += flags[8 + w];
    int total = 0;
    for (int w = 0; w < (NT >> 5); ++w) total += flags[8 + w];
    if (root) cidx[i] = before + __popc(mask & ((1u << lane) - 1u));
    if (i < m) {
      const int l = label[i];
      const int slot = atomicAdd(&memcnt[l], 1);
      if (slot < CSMAX) memb[l * CSMAX + slot] = (unsigned short)i;
    }
    running += total;
    __syncthreads();
  }
  const int ncomp = running;
  {
    int mx = 0;
    for (int i = tid; i < m; i += NT) mx = max(mx, memcnt[i]);
    if (mx > 0) atomicMax(&flags[3], mx);
  }
  __syncthreads();
  const int cs = flags[3];
  if (cs > CSMAX || ncomp * cs > pcap || ncomp * cs * cs > P.wcap || ncomp > 8191) return false;
  st.ncomp = ncomp; st.cs = cs; st.m = m;
  st.sh = 0;
  while ((1 << st.sh) < ncomp) ++st.sh;
  const int npos = ncomp * cs;
  for (int p = tid; p < npos; p += NT) { S.rows()[p] = 0xFFFF; S.ncols()[p] = 0; }
  for (int t = tid; t < ncomp * cs * cs; t += NT) S.Fd()[t] = T(0);
  for (int t = tid; t < UC * pcap; t += NT) { S.Gd()[t] = T(0); S.ccols()[t] = 0; }
  for (int t = tid; t < 8 * ncomp; t += NT) cmap[t] = 0u;
  __syncthreads();
  // ---- rows <-> positions (slot = rank of the row inside its component), column bitmaps
  for (int i = tid; i < m; i += NT) {
    const int l = label[i], c = cidx[l], cnt = memcnt[l];
    int r = 0;
    for (int t = 0; t < cnt; ++t) r += (memb[l * CSMAX + t] < i);
    const int pos = r * ncomp + c;
    S.rows()[pos] = (unsigned short)i;
    S.posof()[i] = (unsigned short)pos;
    const int gc = Gcnt[i];
    for (int k = 0; k < gc; ++k) { const int col = Gi[k * m + i]; atomicOr(&cmap[c * 8 + (col >> 5)], 1u << (col & 31)); }
  }
  __syncthreads();
  // ---- Fd, Gd (slot of a column = its rank in the component's bitmap), sorted column lists
  int bad2 = 0;
  for (int i = tid; i < m; i += NT) {
    const int pos = S.posof()[i], r = pos / ncomp, c = pos - r * ncomp;
    const int fc = Fcnt[i];
    for (int k = 0; k < fc; ++k) {
      const int pj = S.posof()[Fi[k * m + i]];
      S.Fd()[(size_t)(r * cs + pj / ncomp) * ncomp + c] = Fv[k * m + i];
    }
    const int gc = Gcnt[i];
    for (int k = 0; k < gc; ++k) {
      const int col = Gi[k * m + i], wd = col >> 5;
      int p = __popc(cmap[c * 8 + wd] & ((1u << (col & 31)) - 1u));
      for (int w = 0; w < wd; ++w) p += __popc(cmap[c * 8 + w]);
      if (p < UC) { S.Gd()[(size_t)p * pcap + pos] = Gv[k * m + i]; S.ccols()[p * pcap + c] = (unsigned char)col; }
    }
  }
  for (int c = tid; c < ncomp; c += NT) {
    int cnt = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) cnt += __popc(cmap[c * 8 + w]);
    if (cnt > UC) bad2 = 1;
    S.ncols()[c] = (unsigned char)min(cnt, UC);
  }
  if (__syncthreads_or(bad2)) return false;
  // per-column lists of (component, slot): G^T w and the assembly of K gather through them.
  // Filled in arrival order, then ranked (entries are distinct) so that the order is deterministic.
  int bad3 = 0;
  for (int t = tid; t < ncomp * UC; t += NT) {
    const int c = t / UC, p = t - c * UC;
    if (p < S.ncols()[c]) {
      const int a = S.ccols()[p * pcap + c];
      const int slot = atomicAdd(&cl_cnt[a], 1);
      if (slot < LMAX) cl_tmp[slot * n + a] = (unsigned short)(c * 8 + p); else bad3 = 1;
    }
  }
  if (__syncthreads_or(bad3)) return false;
  for (int t = tid; t < n * LMAX; t += NT) {
    const int a = t % n, l = t / n, cnt = cl_cnt[a];
    if (l < cnt) {
      const int v = cl_tmp[l * n + a];
      int rank = 0;
      for (int u = 0; u < cnt; ++u) rank += (cl_tmp[u * n + a] < v);
      S.clist()[rank * n + a] = (unsigned short)v;
    }
    if (l == 0) S.clcnt()[a] = (unsigned char)cnt;
  }
  __syncthreads();
  return true;
}

// ------------------------------------------------------------------ engine path: structure from the contact list
// The fused entry points (lcpb200_engine_forward / _backward) hand the kernels the contact
// structure-of-arrays the engine holds (world.py:139-234, engines.py:50-116) instead of dense Q, G, F:
// the components, their columns and values are known in closed form, nothing dense is read or written.
template <typename T>
struct EngineSoA {
  const T *mass, *inertia, *v, *fext;         // [B,nb] [B,nb] [B,n] [B,n];  mass == nullptr: dense inputs
  const T *normal, *p1, *p2;                  // [B,nc,2]
  const T *mu, *rest;                         // [B,nc]
  const int32_t *b1, *b2;                     // [nc] contact topology, shared by the batch ([B,nc] when nc_s != nullptr)
  const int32_t* nc_s;                        // nullptr, or [B]: contacts of each scene (<= nc; arrays are strided by nc)
  int nb, nc;
  int mode;                                   // 0: solve_dynamics (engines.py:50-76), 1: post_stabilization (engines.py:80-116)
  T dt;
  T *p_s, *h_s;                               // [B,n], [B,m]: p and h of every scene (written here, read by the solver)
};

// Jacobian row of contact c along direction (dx, dy), restricted to the six columns of its two bodies
// (world.py:172-184): body1 gets [p1 x d, d], body2 the negated [p2 x d, d].
template <typename T>
__device__ __forceinline__ void contact_row(T p1x, T p1y, T p2x, T p2y, T dx, T dy, T (&r1)[3], T (&r2)[3]) {
  r1[0] = p1x * dy - p1y * dx; r1[1] = dx; r1[2] = dy;
  r2[0] = -(p2x * dy - p2y * dx); r2[1] = -dx; r2[2] = -dy;
}

template <typename T>
__device__ __noinline__ bool build_structure_soa(const CPlan& P, CSmem<T>& S, Struct& st, const EngineSoA<T>& e_,
                                                 int sc, const T* __restrict__ A, int* singular) {
  const int n = P.n, e = P.e, tid = threadIdx.x, pcap = P.pcap;
  const int nb = e_.nb, ncs = e_.nc, cs = e_.mode == 0 ? 4 : 1;          // ncs: stride of the per-contact arrays
  const int nc = e_.nc_s ? e_.nc_s[sc] : e_.nc;                          // contacts of this scene
  const int m = cs * nc;
  const int32_t* tb1 = e_.b1 + (e_.nc_s ? (size_t)sc * ncs : 0);
  const int32_t* tb2 = e_.b2 + (e_.nc_s ? (size_t)sc * ncs : 0);
  char* sb = reinterpret_cast<char*>(S.K());
  unsigned short* cl_tmp = reinterpret_cast<unsigned short*>(sb);                      // [LMAX][n]
  int* cl_cnt = reinterpret_cast<int*>(sb + al16((size_t)LMAX * n * 2));               // [n]
  if (n != 3 * nb || nc < 0 || nc > ncs || m > P.m || nc * cs > pcap || nc * cs * cs > P.wcap) return false;
  const T* mass = e_.mass + (size_t)sc * nb;
  const T* inertia = e_.inertia + (size_t)sc * nb;
  const T* v = e_.v + (size_t)sc * n;
  const T* normal = e_.normal + (size_t)sc * ncs * 2;
  const T* p1 = e_.p1 + (size_t)sc * ncs * 2;
  const T* p2 = e_.p2 + (size_t)sc * ncs * 2;
  T* ps = e_.p_s + (size_t)sc * n;
  T* hs = e_.h_s + (size_t)sc * P.m;
  int bad = 0;
  for (int j = tid; j < n; j += NT) {
    const int body = j / 3;
    const T q = (j - 3 * body == 0) ? inertia[body] : mass[body];          // world.py:57-61, bodies.py:44-47
    S.qd()[j] = q;
    if (!(q != T(0) && isfinite((double)q))) bad |= 2;
    ps[j] = e_.mode == 0 ? q * v[j] + e_.dt * e_.fext[(size_t)sc * n + j] : T(0);      // engines.py:32 / :109
    cl_cnt[j] = 0;
  }
  for (int t = tid; t < e * n; t += NT) S.As()[t] = A[t];
  st.ncomp = nc; st.cs = cs; st.m = m;
  st.sh = 0;
  while ((1 << st.sh) < nc) ++st.sh;
  for (int t = tid; t < UC * pcap; t += NT) { S.Gd()[t] = T(0); S.ccols()[t] = 0; }
  for (int t = tid; t < nc * cs * cs; t += NT) S.Fd()[t] = T(0);
  __syncthreads();
  for (int c = tid; c < nc; c += NT) {
    const int b1 = tb1[c], b2 = tb2[c];
    if (b1 == b2 || b1 < 0 || b2 < 0 || b1 >= nb) { bad |= 1; continue; }
    // b2 >= nb: a static obstacle (no dofs). The contact's rows touch body1's three columns only.
    const bool two = b2 < nb;
    const int lo = two ? min(b1, b2) : b1, hi = max(b1, b2);
    const int o1 = b1 < b2 ? 0 : 3, o2 = 3 - o1;                   // slots of body1 / body2 in the sorted column list
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      S.ccols()[q * pcap + c] = (unsigned char)(3 * lo + q);
      if (two) S.ccols()[(3 + q) * pcap + c] = (unsigned char)(3 * hi + q);
    }
    S.ncols()[c] = two ? 6 : 3;
    const T nx = normal[2 * c], ny = normal[2 * c + 1];
    const T p1x = p1[2 * c], p1y = p1[2 * c + 1], p2x = p2[2 * c], p2y = p2[2 * c + 1];
    T r1[3], r2[3];
    contact_row<T>(p1x, p1y, p2x, p2y, nx, ny, r1, r2);            // Jc row
    const T v20 = two ? v[3 * b2] : T(0), v21 = two ? v[3 * b2 + 1] : T(0), v22 = two ? v[3 * b2 + 2] : T(0);
    const T jv = r1[0] * v[3 * b1] + r1[1] * v[3 * b1 + 1] + r1[2] * v[3 * b1 + 2] +
                 r2[0] * v20 + r2[1] * v21 + r2[2] * v22;
    const T rc = e_.rest[(size_t)sc * ncs + c];
#pragma unroll
    for (int q = 0; q < 3; ++q) { S.Gd()[(size_t)(o1 + q) * pcap + c] = r1[q]; if (two) S.Gd()[(size_t)(o2 + q) * pcap + c] = r2[q]; }
    S.rows()[c] = (unsigned short)c;
    S.posof()[c] = (unsigned short)c;
    if (e_.mode == 0) {
      hs[c] = jv * rc;                                             // engines.py:53,74
      contact_row<T>(p1x, p1y, p2x, p2y, ny, -nx, r1, r2);         // Jf rows: +- left_orthogonal(n)  (world.py:186-211)
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        S.Gd()[(size_t)(o1 + q) * pcap + nc + c] = r1[q];
        S.Gd()[(size_t)(o1 + q) * pcap + 2 * nc + c] = -r1[q];
        if (two) { S.Gd()[(size_t)(o2 + q) * pcap + nc + c] = r2[q]; S.Gd()[(size_t)(o2 + q) * pcap + 2 * nc + c] = -r2[q]; }
      }
      const int rw[4] = {c, nc + 2 * c, nc + 2 * c + 1, 3 * nc + c};
#pragma unroll
      for (int r = 0; r < 4; ++r) { S.rows()[r * nc + c] = (unsigned short)rw[r]; S.posof()[rw[r]] = (unsigned short)(r * nc + c); }
      hs[nc + 2 * c] = T(0); hs[nc + 2 * c + 1] = T(0); hs[3 * nc + c] = T(0);
      // F = [[0,0,0],[0,0,E],[mu,-E^T,0]]  (engines.py:69-73): rows/cols {c, f1, f2, gamma} of the component
      S.Fd()[(size_t)(1 * 4 + 3) * nc + c] = T(1);
      S.Fd()[(size_t)(2 * 4 + 3) * nc + c] = T(1);
      S.Fd()[(size_t)(3 * 4 + 0) * nc + c] = e_.mu[(size_t)sc * ncs + c];
      S.Fd()[(size_t)(3 * 4 + 1) * nc + c] = T(-1);
      S.Fd()[(size_t)(3 * 4 + 2) * nc + c] = T(-1);
    } else {
      hs[c] = jv + jv * -rc;                                       // engines.py:90
    }
    // column lists: arrival order, ranked below
    for (int q = 0; q < (two ? 6 : 3); ++q) {
      const int a = q < 3 ? 3 * lo + q : 3 * hi + q - 3;
      const int slot = atomicAdd(&cl_cnt[a], 1);
      if (slot < LMAX) cl_tmp[slot * n + a] = (unsigned short)(c * 8 + q); else bad |= 1;
    }
  }
  const int anybad = __syncthreads_or(bad);
  if (anybad & 2) { *singular = 1; return false; }
  if (anybad & 1) return false;
  for (int t = tid; t < n * LMAX; t += NT) {
    const int a = t % n, l = t / n, cnt = cl_cnt[a];
    if (l < cnt) {
      const int val = cl_tmp[l * n + a];
      int rank = 0;
      for (int u = 0; u < cnt; ++u) rank += (cl_tmp[u * n + a] < val);
      S.clist()[rank * n + a] = (unsigned short)val;
    }
    if (l == 0) S.clcnt()[a] = (unsigned char)cnt;
  }
  __syncthreads();
  return true;
}

// Which LU factors this scene's K (factor_kkt). Block (i, j) of K = Q + G^T W G (16 x 16 blocks) is non-zero only
// when one component of G has columns in both blocks, so the block band of K is the widest spread of a component's
// sorted column list, and an LU without pivoting keeps it. Equality rows border K with A, which couples every
// block: such scenes take the dense LU, as do all scenes under CFLAG_DENSE_LU. Called by the whole CTA once the
// column lists are in shared memory; thread 0 writes the answer, the barrier before the scene's first
// factorisation publishes it.
template <typename T>
__device__ __noinline__ void mark_band_lu(const CPlan& P, CSmem<T> S, Struct st) {
  int wide = P.e > 0 || (P.flags & CFLAG_DENSE_LU);
  for (int c = threadIdx.x; c < st.ncomp; c += NT) {
    const int nc = S.ncols()[c];
    if (nc > 0 && (S.ccols()[(nc - 1) * P.pcap + c] >> 4) - (S.ccols()[c] >> 4) > LU_BW) wide = 1;
  }
  wide = __syncthreads_or(wide);
  if (threadIdx.x == 0) S.misc()[MISC_BAND_LU] = !wide;
}

__device__ __forceinline__ double rcp64_fast(double x) {
  // MUFU.RCP64H seed (>= 20 bits) + 2 Newton steps; exact division outside the seed's range
  double r;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
  const double ax = fabs(x);
  if (!(ax > 1e-290 && ax < 1e290)) return 1.0 / x;
  r = fma(r, fma(-x, r, 1.0), r);
  r = fma(r, fma(-x, r, 1.0), r);
  return r;
}

// ------------------------------------------------------------------ W_c = (Fd_c + diag(1/d))^-1
// One thread per component: in-place Gauss-Jordan with partial pivoting, the block held in
// registers (static indices only: row interchanges are conditional swaps, recorded in a bit mask and
// undone as column swaps in reverse order at the end). Slot-major arrays: thread c reads / writes
// consecutive addresses (no bank conflicts).
template <typename T, int CS>
__device__ __forceinline__ void comp_inverse(const CPlan& P, CSmem<T>& S, const Struct& st) {
  const int nc_ = st.ncomp;                       // positions are slot-major: pos(c, r) = r * ncomp + c
  for (int c = threadIdx.x; c < nc_; c += NT) {
    double M[CS][CS];
#pragma unroll
    for (int r = 0; r < CS; ++r) {
      const int i = S.rows()[r * nc_ + c];
#pragma unroll
      for (int q = 0; q < CS; ++q) M[r][q] = (double)S.Fd()[(size_t)(r * CS + q) * nc_ + c];
      M[r][r] += (i == 0xFFFF) ? 1.0 : ((P.flags & 1) ? 1.0 / (double)S.d()[i] : (double)(T(1) / S.d()[i]));      // 1/d in the I/O dtype (pdipm.py:427-429)
    }
    unsigned swaps = 0;
    int bit = 0;
#pragma unroll
    for (int k = 0; k < CS; ++k) {
#pragma unroll
      for (int i = k + 1; i < CS; ++i) {           // bring the largest |M[i][k]|, i >= k, to row k
        const bool sw = fabs(M[i][k]) > fabs(M[k][k]);
        swaps |= (sw ? 1u : 0u) << bit;
        ++bit;
#pragma unroll
        for (int q = 0; q < CS; ++q) { const double u = M[k][q], w = M[i][q]; M[k][q] = sw ? w : u; M[i][q] = sw ? u : w; }
      }
      const double r = rcp64_fast(M[k][k]);
      M[k][k] = 1.0;
#pragma unroll
      for (int q = 0; q < CS; ++q) M[k][q] *= r;
#pragma unroll
      for (int i = 0; i < CS; ++i) {
        if (i == k) continue;
        const double f = M[i][k];
        M[i][k] = 0.0;
#pragma unroll
        for (int q = 0; q < CS; ++q) M[i][q] = fma(-f, M[k][q], M[i][q]);
      }
    }
#pragma unroll
    for (int k = CS - 1; k >= 0; --k) {
#pragma unroll
      for (int i = CS - 1; i > k; --i) {
        --bit;
        const bool sw = (swaps >> bit) & 1u;
#pragma unroll
        for (int q = 0; q < CS; ++q) { const double u = M[q][k], w = M[q][i]; M[q][k] = sw ? w : u; M[q][i] = sw ? u : w; }
      }
    }
#pragma unroll
    for (int r = 0; r < CS; ++r)
#pragma unroll
      for (int q = 0; q < CS; ++q) S.W()[(size_t)(r * CS + q) * nc_ + c] = M[r][q];
  }
}

// Positions per thread comp_apply needs for rows of CS slots: the grid it covers is t < CS << sh, sh = ceil(log2(ncomp)).
// build_structure admits ncomp * CS <= pcap <= 4 NT (pcap is m rounded up to 8, m <= 4 NT), so ncomp <= 4 NT / CS:
// 4 for CS = 1, 2, 4; 5 for CS = 5 (ncomp <= 204: 5 << 8 = 1280); 6 for CS = 3 (ncomp <= 341: 3 << 9) and 6 (ncomp <= 170).
template <int CS>
struct ApplySpan {
  static constexpr int ceil_log2(int x) { return x <= 1 ? 0 : 1 + ceil_log2((x + 1) / 2); }
  static constexpr int U = ((CS << ceil_log2(4 * NT / CS)) + NT - 1) / NT;
};

// out_c = W_c * in_c for every component, in place in S.scr (one thread per (component, row))
template <typename T, int CS>
__device__ __forceinline__ void comp_apply(CSmem<T>& S, const Struct& st, bool trans = false) {
  constexpr int U = ApplySpan<CS>::U;
  const int nc_ = st.ncomp;                       // positions are slot-major: pos(c, r) = r * ncomp + c
  const int npos = nc_ * CS;
  const int sh = st.sh, cmask = (1 << sh) - 1, tot = CS << sh;
  double val[U];
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const int t = threadIdx.x + u * NT, r = t >> sh, c = t & cmask;
    val[u] = 0.0;
    if (t < tot && c < nc_) {
      double a = 0.0;
#pragma unroll
      for (int q = 0; q < CS; ++q) a = fma(S.W()[(size_t)(trans ? (q * CS + r) : (r * CS + q)) * nc_ + c], S.scr()[q * nc_ + c], a);
      val[u] = a;
    }
  }
  __syncthreads();
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const int t = threadIdx.x + u * NT, r = t >> sh, c = t & cmask;
    if (t < tot && c < nc_) S.scr()[r * nc_ + c] = val[u];
  }
  (void)npos;
}

// ------------------------------------------------------------------ K (column major, fp64)
// Kbar = [[Q + G^T W G, A^T], [A, 0]] padded with an identity block to NP. A group of UC = 8 lanes
// owns one row a of K: lane q2 of the group adds the contribution of list entry l (component c, slot
// p of column a) to K[a][column q2 of c]; the groups walk their lists in lockstep (__syncwarp
// between entries), so every entry of K is accumulated in list order -- deterministic, no atomics.
template <typename T, int NS, int CS>
__device__ __forceinline__ void assemble_K(const CPlan& P, CSmem<T>& S, const Struct& st) {
  const int nc_ = st.ncomp;                       // positions are slot-major: pos(c, r) = r * ncomp + c
  constexpr int NP = 16 * NS;
  const int n = P.n, N = P.N, e = P.e, tid = threadIdx.x, pcap = P.pcap;
  double* K = S.K();
  {
    double2* K2 = reinterpret_cast<double2*>(K);
    for (int t = tid; t < NP * NP / 2; t += NT) K2[t] = make_double2(0.0, 0.0);
  }
  __syncthreads();
  for (int i = tid; i < NP; i += NT) K[(size_t)i * NP + i] = i < n ? (double)S.qd()[i] : (i < N ? 0.0 : 1.0);
  for (int t = tid; t < e * n; t += NT) {
    const int k = t / n, i = t - k * n;
    const double v = (double)S.As()[t];
    K[(size_t)(n + k) * NP + i] = v;                 // A^T: K[i][n+k]
    K[(size_t)i * NP + n + k] = v;                   // A  : K[n+k][i]
  }
  __syncthreads();
  const int grp = tid >> 3, q2 = tid & 7;            // 32 groups of 8 lanes
  for (int a0 = 0; a0 < n; a0 += NT / 8) {
    const int a = a0 + grp;
    const int cnt = a < n ? (int)S.clcnt()[a] : 0;
    int mx = cnt;                                    // warp-uniform trip count (4 groups per warp)
    mx = max(mx, __shfl_xor_sync(FULL, mx, 8));
    mx = max(mx, __shfl_xor_sync(FULL, mx, 16));
    for (int l = 0; l < mx; ++l) {
      if (l < cnt) {
        const int cp = S.clist()[l * n + a], c = cp >> 3, p = cp & 7;
        if (q2 < (int)S.ncols()[c]) {
          double acc = 0.0;
#pragma unroll
          for (int q = 0; q < CS; ++q) {             // u_q = sum_r Gd[r][p] W[r][q];  acc += u_q Gd[q][q2]
            double u = 0.0;
#pragma unroll
            for (int r = 0; r < CS; ++r)
              u = fma((double)S.Gd()[(size_t)p * pcap + r * nc_ + c], S.W()[(size_t)(r * CS + q) * nc_ + c], u);
            acc = fma(u, (double)S.Gd()[(size_t)q2 * pcap + q * nc_ + c], acc);
          }
          K[(size_t)S.ccols()[q2 * pcap + c] * NP + a] += acc;
        }
      }
      __syncwarp();
    }
  }
  __syncthreads();
}

// ------------------------------------------------------------------ LU in registers
// Thread (ti = tid & 15, tj = tid >> 4) owns a[r][c] = K[16r + ti][16c + tj]. One phase = the 16
// pivots of block B0, two per barrier. Pivot rows / columns travel through shared memory as
// interleaved pairs (U2[j] = {row k, row k+1} at column j, C2[i] = {column k, column k+1} at row i,
// double buffered); every thread redoes the 2x2 pivot arithmetic. No pivoting: K + its border is
// quasi-definite; zero pivots produce inf/nan exactly like the reference's LU would.
// The loop is bound by the FP64 pipe (16 lanes / SMSP): masks are applied only in the diagonal
// block's slots, and the two column passes keep the live registers under the 128 of 2 CTAs / SM.
//
// Block band BW < NS - 1: the thread holds only the blocks with |r - c| <= BW, and phase B0 loads and
// updates only blocks r, c in [B0, B0 + BW]. That is exact for a K whose non-zero blocks lie in the
// band (mark_band_lu): without pivoting, the pivot rows and columns of phase B0 are zero beyond block
// B0 + BW, so there the dense form adds products of a zero and a finite value, which leave every entry
// as it was (K holds no -0). The entries that are computed see the same operations in the same order as
// in the dense form: the factors are bitwise the same unless a pivot is zero or not finite.
template <int NS, int BW>
struct LuBand {
  static constexpr bool DENSE = BW >= NS - 1;
  static constexpr int W = DENSE ? NS : 2 * BW + 1;             // block columns held per block row
  static __device__ __forceinline__ constexpr bool in(int r, int c) { return DENSE || (r - c <= BW && c - r <= BW); }
  static __device__ __forceinline__ constexpr int col(int r, int c) { return DENSE ? c : c - r + BW; }   // slot of block (r, c)
  static __host__ __device__ constexpr int end(int b0) { return DENSE || b0 + BW + 1 > NS ? NS : b0 + BW + 1; }   // phase b0: [b0, end)
};

template <int NS, int BW, int B0>
__device__ __forceinline__ void lu_phase(double (&a)[NS][LuBand<NS, BW>::W], int o_buf, int o_rdiag, int& step, int ti,
                                         int tj) {
  // Entries keep the value they had when their column became the pivot column: after the last
  // phase a[i][j] (i > j) = u_jj L[i][j] and a[i][j] (i <= j) = U[i][j]; factor_K scales by 1/u_jj.
  // With that convention a step is ONE masked rank-2 update, a -= m0 (x) w0 + m1 (x) w1, with
  //   m0_i = [i > k] a_ik / a_kk,             w0_j = [j > k] a_kj,
  //   m1_i = [i > k+1] (a_i,k+1 - m0_i a_k,k+1) / a'_k+1,k+1,   w1_j = [j > k+1] (a_k+1,j - l10 a_kj),
  // and the masks only matter inside the diagonal block (r == B0 / c == B0).
  using Bd = LuBand<NS, BW>;
  constexpr int NP = 16 * NS;
  constexpr int E = Bd::end(B0);
  constexpr int L = E - B0;                           // live block rows / columns
  constexpr int CW = (L <= 4) ? L : 3;                // columns per pass (bounds the live registers)
  double* const rdiag = reinterpret_cast<double*>(cnd_smem + o_rdiag);
#pragma unroll 1
  for (int kk = 0; kk < 16; kk += 2) {
    const int k = 16 * B0 + kk;
    double2* const U2 = reinterpret_cast<double2*>(cnd_smem + o_buf) + (size_t)(step & 1) * 2 * NP;
    double2* const C2 = U2 + NP;
    ++step;
    {
      const int sr = ti - kk, sc = tj - kk;
      if ((unsigned)sr < 2u) {                        // I hold part of pivot row k (sr = 0) or k+1 (sr = 1)
        double* dst = reinterpret_cast<double*>(U2) + sr;
#pragma unroll
        for (int c = B0; c < E; ++c) dst[2 * (16 * c + tj)] = a[B0][Bd::col(B0, c)];
      }
      if ((unsigned)sc < 2u) {                        // ... of pivot column k / k+1
        double* dst = reinterpret_cast<double*>(C2) + sc;
#pragma unroll
        for (int r = B0; r < E; ++r) dst[2 * (16 * r + ti)] = a[r][Bd::col(r, B0)];
      }
    }
    __syncthreads();
    const double2 pk = U2[k], pk1 = U2[k + 1];        // pk = {a_kk, a_k+1,k}, pk1 = {a_k,k+1, a_k+1,k+1}
    // 1/a_kk and 1/a'_k+1,k+1 = a_kk / det(2x2 pivot block): two independent reciprocals
    const double p01 = pk1.x;
    const double r0 = rcp64_fast(pk.x);
    const double r1 = pk.x * rcp64_fast(fma(pk.x, pk1.y, -(pk.y * p01)));
    const double l10 = pk.y * r0;
    if ((ti | tj) == 0) { rdiag[k] = r0; rdiag[k + 1] = r1; }
#pragma unroll
    for (int cg = B0; cg < E; cg += CW) {
      double w0[CW], w1[CW];                          // pivot rows restricted to this pass's columns
#pragma unroll
      for (int q = 0; q < CW; ++q) {
        const int c = cg + q;
        if (c < E) {
          const double2 u = U2[16 * c + tj];
          const double x1 = fma(-l10, u.x, u.y);
          w0[q] = (c == B0 && !(tj > kk)) ? 0.0 : u.x;
          w1[q] = (c == B0 && !(tj > kk + 1)) ? 0.0 : x1;
        }
      }
#pragma unroll
      for (int r = B0; r < E; ++r) {
        const double2 cc = C2[16 * r + ti];
        double m0 = cc.x * r0;
        double m1 = fma(-m0, p01, cc.y) * r1;
        if (r == B0) {
          m0 = (ti > kk) ? m0 : 0.0;
          m1 = (ti > kk + 1) ? m1 : 0.0;
        }
#pragma unroll
        for (int q = 0; q < CW; ++q) {
          const int c = cg + q;
          if (c < E) a[r][Bd::col(r, c)] = fma(-m1, w1[q], fma(-m0, w0[q], a[r][Bd::col(r, c)]));
        }
      }
    }
  }
}

template <int NS, int BW, int B0>
struct LuPhases {
  static __device__ __forceinline__ void run(double (&a)[NS][LuBand<NS, BW>::W], int o_buf, int o_rdiag, int& step, int ti,
                                             int tj) {
    lu_phase<NS, BW, B0>(a, o_buf, o_rdiag, step, ti, tj);
    LuPhases<NS, BW, B0 + 1>::run(a, o_buf, o_rdiag, step, ti, tj);
  }
};
template <int NS, int BW>
struct LuPhases<NS, BW, NS> {
  static __device__ __forceinline__ void run(double (&)[NS][LuBand<NS, BW>::W], int, int, int&, int, int) {}
};

// Layout of the factors for the substitution warp (solve_warp): lane l owns rows QN*l + q', round
// r eliminates the QN pivots QN*r + q; entry (i, j) sits at
//     ((r_j * QN + q'_i) * QN + q_j) * 32 + lane_i
// so that each (q', q) pair of a round is one conflict-free 8-byte load per lane. L[i][j] for
// i > j, U[i][j] / u_jj for i < j (the diagonal slots are unused); both are a[i][j] / u_jj.
template <int NS> struct SolveLayout {
  static constexpr int NP = 16 * NS;
  static constexpr int QN = (NP + 31) / 32;
  static constexpr int ROUNDS = NP / QN;
  static constexpr size_t BYTES = (size_t)ROUNDS * QN * QN * 32 * 8;
};

// K (shared, column major) -> registers -> LU -> factors back to the K region in the solve layout.
// BW = NS - 1: dense; BW < NS - 1: only the block band |r - c| <= BW of K is non-zero (LuBand).
template <int NS, int BW>
__device__ __forceinline__ void factor_K_body(int o_K, int o_rdiag, bool trans) {
  using Bd = LuBand<NS, BW>;
  constexpr int NP = 16 * NS, QN = SolveLayout<NS>::QN;
  int tid_;                                          // read %tid.x once (opaque to the compiler: no re-reads in the loops)
  asm volatile("mov.u32 %0, %%tid.x;" : "=r"(tid_));
  const int ti = tid_ & 15, tj = tid_ >> 4;
  double* const K = reinterpret_cast<double*>(cnd_smem + o_K);
  double* const rdiag = reinterpret_cast<double*>(cnd_smem + o_rdiag);
  double a[NS][Bd::W];
#pragma unroll
  for (int c = 0; c < NS; ++c)
#pragma unroll
    for (int r = 0; r < NS; ++r)
      if (Bd::in(r, c)) a[r][Bd::col(r, c)] = K[(size_t)(16 * c + tj) * NP + 16 * r + ti];
  __syncthreads();                                   // K region becomes the broadcast buffer
  int step = 0;
  LuPhases<NS, BW, 0>::run(a, o_K, o_rdiag, step, ti, tj);
  __syncthreads();                                   // rdiag complete, broadcast buffers dead
  // trans (exact-adjoint backward): K^T = U^T L^T = L' U' with L'[i][k] = U[k][i] / u_kk and
  // U'[i][k] / u'_kk = u_ii L[k][i] / u_kk, i.e. entry (i, k) of the solve layout receives a[k][i] / u_kk:
  // the roles of the row and column index of a are swapped, the scale is the ROW's reciprocal pivot.
  int rowpart[NS];
  double rrow[NS];
#pragma unroll
  for (int r = 0; r < NS; ++r) {
    const int i = 16 * r + ti;
    rowpart[r] = trans ? (i / QN) * QN * QN * 32 + (i % QN) * 32 : (i % QN) * QN * 32 + i / QN;
    rrow[r] = rdiag[i];
  }
#pragma unroll
  for (int c = 0; c < NS; ++c) {
    const int j = 16 * c + tj;
    const double rj = rdiag[j];
    const int colpart = trans ? (j % QN) * QN * 32 + j / QN : (j / QN) * QN * QN * 32 + (j % QN) * 32;
#pragma unroll
    for (int r = 0; r < NS; ++r) {
      const int i = 16 * r + ti;
      // out of the band the dense LU leaves +0 and scales it like any other entry: write the same product
      // (the region still holds K there)
      const double v = Bd::in(r, c) ? a[r][Bd::col(r, c)] : 0.0;
      K[colpart + rowpart[r]] = (i != j) ? v * (trans ? rrow[r] : rj) : v;
    }
  }
  __syncthreads();
}

// One call target for both LU variants: with two, ptxas saved more of the callers' registers around the dense LU
// (double, NS = 6 forward: 16 / 40 B of spills in the dense LU became 48 / 88 B).
template <int NS>
__device__ __noinline__ void factor_K(int o_K, int o_rdiag, bool trans, bool band) {
  if constexpr (LU_BW < NS - 1) {
    if (band) {
      factor_K_body<NS, LU_BW>(o_K, o_rdiag, trans);
      return;
    }
  }
  factor_K_body<NS, NS - 1>(o_K, o_rdiag, trans);
}

// ------------------------------------------------------------------ triangular solves (ONE warp)
// bx <- Kbar^-1 bx. Exact substitution order; the QN pivots of a round belong to ONE lane (rows
// QN*r .. QN*r + QN-1 of lane r), are broadcast by shuffles, their QN x QN triangular piece is
// solved redundantly by every lane, then each lane updates its own rows. The coefficients of
// round r+1 are loaded while round r's dependent chain runs (software pipeline, two register
// sets), and the row update is predicated, not branched: the chain per round is one 64-bit shuffle
// (26 cycles) + QN dependent DFMAs (8 cycles each).
template <int QN>
struct SolveCoef {
  double dg[QN * QN];         // lane r's slots (the pivots' own triangular piece), broadcast
  double rw[QN * QN];         // this lane's slots
};

template <int QN>
__device__ __forceinline__ void solve_load(SolveCoef<QN>& c, const double* blk, int r, int lane) {
#pragma unroll
  for (int t = 0; t < QN * QN; ++t) { c.dg[t] = blk[t * 32 + r]; c.rw[t] = blk[t * 32 + lane]; }
}

template <int QN>
__device__ __forceinline__ void solve_round_fwd(double (&y)[QN], const SolveCoef<QN>& c, int r, int lane) {
  double v[QN];
#pragma unroll
  for (int q = 0; q < QN; ++q) v[q] = __shfl_sync(FULL, y[q], r);
#pragma unroll
  for (int q = 0; q < QN; ++q)
#pragma unroll
    for (int qp = q + 1; qp < QN; ++qp) v[qp] = fma(-c.dg[qp * QN + q], v[q], v[qp]);
  const bool below = lane > r, own = lane == r;
#pragma unroll
  for (int qp = 0; qp < QN; ++qp) {
    double t = y[qp];
#pragma unroll
    for (int q = 0; q < QN; ++q) t = fma(-c.rw[qp * QN + q], v[q], t);
    y[qp] = below ? t : (own ? v[qp] : y[qp]);
  }
}

template <int QN>
__device__ __forceinline__ void solve_round_bwd(double (&y)[QN], const SolveCoef<QN>& c, int r, int lane) {
  double v[QN];
#pragma unroll
  for (int q = 0; q < QN; ++q) v[q] = __shfl_sync(FULL, y[q], r);
#pragma unroll
  for (int q = QN - 1; q >= 0; --q)
#pragma unroll
    for (int qp = q - 1; qp >= 0; --qp) v[qp] = fma(-c.dg[qp * QN + q], v[q], v[qp]);
  const bool above = lane < r, own = lane == r;
#pragma unroll
  for (int qp = 0; qp < QN; ++qp) {
    double t = y[qp];
#pragma unroll
    for (int q = QN - 1; q >= 0; --q) t = fma(-c.rw[qp * QN + q], v[q], t);
    y[qp] = above ? t : (own ? v[qp] : y[qp]);
  }
}

template <int NS>
__device__ __noinline__ void solve_warp(int o_K, int o_rdiag, int o_bx) {
  constexpr int NP = 16 * NS, QN = SolveLayout<NS>::QN, ROUNDS = SolveLayout<NS>::ROUNDS;
  constexpr int STRIDE = QN * QN * 32;
  static_assert(ROUNDS % 2 == 0, "the software pipeline handles two rounds per trip");
  const int lane = threadIdx.x & 31;
  const double* const S = reinterpret_cast<const double*>(cnd_smem + o_K);
  const double* const rdiag = reinterpret_cast<const double*>(cnd_smem + o_rdiag);
  double* const bx = reinterpret_cast<double*>(cnd_smem + o_bx);
  double y[QN];
#pragma unroll
  for (int q = 0; q < QN; ++q) y[q] = (QN * lane + q < NP) ? bx[QN * lane + q] : 0.0;
  SolveCoef<QN> c0, c1;
  // ---- forward: L y = b (unit lower)
  solve_load<QN>(c0, S, 0, lane);
#pragma unroll 1
  for (int r = 0; r < ROUNDS; r += 2) {
    solve_load<QN>(c1, S + (size_t)(r + 1) * STRIDE, r + 1, lane);
    solve_round_fwd<QN>(y, c0, r, lane);
    const int rn = (r + 2 < ROUNDS) ? r + 2 : ROUNDS - 1;       // last trip: a harmless reload
    solve_load<QN>(c0, S + (size_t)rn * STRIDE, rn, lane);
    solve_round_fwd<QN>(y, c1, r + 1, lane);
  }
  // ---- backward: U x = y with the columns of U pre-scaled by 1/u_kk (z_k = u_kk x_k)
  // (c0 holds round ROUNDS-1 from the last trip above)
#pragma unroll 1
  for (int r = ROUNDS - 1; r > 0; r -= 2) {
    solve_load<QN>(c1, S + (size_t)(r - 1) * STRIDE, r - 1, lane);
    solve_round_bwd<QN>(y, c0, r, lane);
    const int rn = (r - 2 >= 0) ? r - 2 : 0;
    solve_load<QN>(c0, S + (size_t)rn * STRIDE, rn, lane);
    solve_round_bwd<QN>(y, c1, r - 1, lane);
  }
#pragma unroll
  for (int q = 0; q < QN; ++q) {
    const int i = QN * lane + q;
    if (i < NP) bx[i] = y[q] * rdiag[i];
  }
}

// ------------------------------------------------------------------ solve_kkt (pdipm.py:325-354)
// Inputs (nullptr == zero vector): rx[n], rs[m], rz[m], ry[e]; outputs dx[n], ds[m], dz[m], dy[e].
// solve_kkt, factor_kkt and the phases of forward_scene are __noinline__: each one recomputes its addresses from
// the kernel parameters, so that nothing but a few loop scalars is live across the factorisation and the
// substitution (whose register budget is the whole 128 of two CTAs per SM). Spilled values would live in local
// memory, and with ~220 KB of shared memory per SM the L1 left for it is too small: a reload is an L2 round trip.
template <typename T, int CS, int NS, typename PF>
__device__ __noinline__ void solve_kkt(const CPlan& P, CSmem<T> S, Struct st, PF& pf, const T* rx,
                                       const T* rs, const T* rz, const T* ry, T* dx, T* ds, T* dz, T* dy,
                                       bool trans = false) {
  const int nc_ = st.ncomp;                       // positions are slot-major: pos(c, r) = r * ncomp + c
  const int n = P.n, e = P.e, N = P.N, NP = P.NP, tid = threadIdx.x, pcap = P.pcap;
  const int npos = st.ncomp * CS;
  // t = rz - rs/d  -> v = W t
  for (int p = tid; p < npos; p += NT) {
    const int i = S.rows()[p];
    double t = 0.0;
    if (i != 0xFFFF) t = (P.flags & 2) ? ((double)(rz ? rz[i] : T(0)) - (double)rs[i] / (double)S.d()[i]) : (double)((rz ? rz[i] : T(0)) - rs[i] / S.d()[i]);
    S.scr()[p] = t;
  }
  __syncthreads();
  comp_apply<T, CS>(S, st, trans);
  __syncthreads();
  for (int a = tid; a < NP; a += NT) {
    double acc = 0.0;
    if (a < n) {
      const int cnt = S.clcnt()[a];
      for (int l = 0; l < cnt; ++l) {
        const int cp = S.clist()[l * n + a], c = cp >> 3, p = cp & 7;
#pragma unroll
        for (int r = 0; r < CS; ++r) acc = fma((double)S.Gd()[(size_t)p * pcap + r * nc_ + c], S.scr()[r * nc_ + c], acc);
      }
      acc = -(double)(rx ? rx[a] : T(0)) - acc;
    } else if (a < N) {
      acc = -(double)(ry ? ry[a - n] : T(0));
    }
    S.bx()[a] = acc;
  }
  __syncthreads();
  pf.lap(CPH_SOLVE_RHS);
  if (tid < 32) solve_warp<NS>(P.o_K, P.o_rdiag, P.o_bx);
  __syncthreads();
  pf.lap(CPH_SOLVE_TRI);
  // dz = W (G dx + t)
  for (int tt = tid; tt < (CS << st.sh); tt += NT) {
    const int c = tt & ((1 << st.sh) - 1);
    if (c >= nc_) continue;
    const int p = (tt >> st.sh) * nc_ + c;
    const int i = S.rows()[p];
    double t = 0.0;
    if (i != 0xFFFF) {
      const int nc = S.ncols()[c];
      t = (P.flags & 2) ? ((double)(rz ? rz[i] : T(0)) - (double)rs[i] / (double)S.d()[i]) : (double)((rz ? rz[i] : T(0)) - rs[i] / S.d()[i]);
      for (int q = 0; q < nc; ++q) t = fma((double)S.Gd()[(size_t)q * pcap + p], S.bx()[S.ccols()[q * pcap + c]], t);
    }
    S.scr()[p] = t;
  }
  __syncthreads();
  comp_apply<T, CS>(S, st, trans);
  __syncthreads();
  for (int p = tid; p < npos; p += NT) {
    const int i = S.rows()[p];
    if (i == 0xFFFF) continue;
    const T wz = (T)S.scr()[p];
    const T rsi = rs[i];                                         // (dz may alias rs)
    dz[i] = wz;                                                  // :351
    ds[i] = (-rsi - wz) / S.d()[i];                                // :347,350
  }
  for (int a = tid; a < n; a += NT) dx[a] = (T)S.bx()[a];
  for (int k = tid; k < e; k += NT) dy[k] = (T)S.bx()[n + k];
  __syncthreads();
  pf.lap(CPH_SOLVE_POST);
}

// d is in S.d(): W, K, LU
template <typename T, int NS, int CS, typename PF>
__device__ __noinline__ void factor_kkt(const CPlan& P, CSmem<T> S, Struct st, PF& pf, bool trans = false) {
  comp_inverse<T, CS>(P, S, st);
  __syncthreads();
  pf.lap(CPH_WINV);
  assemble_K<T, NS, CS>(P, S, st);
  pf.lap(CPH_ASSEMBLE);
  if constexpr (LU_BW < NS - 1) factor_K<NS>(P.o_K, P.o_rdiag, trans, S.misc()[MISC_BAND_LU] != 0);
  else factor_K<NS>(P.o_K, P.o_rdiag, trans, false);
  pf.lap(CPH_LU);
}

// ------------------------------------------------------------------ get_step (pdipm.py:182-186), per scene
// a = -v/dv; entries with dv > 0 are replaced by max(1, max(a)) (the maximum over ALL entries),
// then the row minimum. One fused block reduction: max(a), min over the entries that are not
// replaced, and whether any entry is replaced; torch NaN semantics (NaN wins min/max; python's
// max(1.0, nan) is 1.0).
template <typename T>
__device__ __forceinline__ void get_steps(const T* z, const T* dz, const T* s, const T* ds, int m, T* red, T& step_z,
                                          T& step_s) {
  const T NEG_INF = -INFINITY, POS_INF = INFINITY;
  T mx[2] = {NEG_INF, NEG_INF};
  T mn[2] = {POS_INF, POS_INF};
  T any[2] = {T(0), T(0)};
  for (int i = threadIdx.x; i < m; i += NT) {
    const T az = -z[i] / dz[i], as = -s[i] / ds[i];
    mx[0] = nan_max(mx[0], az);
    mx[1] = nan_max(mx[1], as);
    if (dz[i] > T(0)) any[0] = T(1); else mn[0] = nan_min(mn[0], az);
    if (ds[i] > T(0)) any[1] = T(1); else mn[1] = nan_min(mn[1], as);
  }
  T v[6] = {mx[0], mx[1], -mn[0], -mn[1], any[0], any[1]};     // min(x) = -max(-x): one reduction operator
  block_reduce<T, 6>(v, OpMax(), NEG_INF, red);
  const T fz = (v[0] > T(1)) ? v[0] : T(1);                     // python max(1.0, a.max()): NaN -> 1.0
  const T fs = (v[1] > T(1)) ? v[1] : T(1);
  step_z = (v[4] > T(0)) ? nan_min(-v[2], fz) : -v[2];
  step_s = (v[5] > T(0)) ? nan_min(-v[3], fs) : -v[3];
}

template <typename T>
struct CFwdArgs {
  CPlan P;
  int B;
  const T *Q, *p, *G, *h, *A, *b, *F;
  T *zhat, *nu, *lam, *slack, *resid;
  int *status, *iters;
  T eps;
  int not_improved_lim, max_iter;
  long long* prof;            // nullptr or [grid][CPH_COUNT]
  EngineSoA<T> soa;           // soa.mass != nullptr: structure, p and h come from the contact list (Q, G, F unused)
  unsigned char* ssave;       // nullptr or [B][P.sbytes]: the structure found for every scene, kept for the backward
};

template <typename T>
struct CBwdArgs {
  CPlan P;
  int B;
  // R cotangents per scene: g and every gradient output are [R][B][...], slot r of scene sc at row r B + sc.
  // A work item is (scene, chunk): chunk k of `chunks` factors the scene's KKT matrix once and solves for the
  // cotangents [R k / chunks, R (k + 1) / chunks).
  int R, chunks;
  const T *Q, *G, *A, *F;
  const T *zhat, *nu, *lam, *slack, *g;
  T *dQ, *dp, *dG, *dh, *dA, *db, *dF;
  int* done;                  // nullptr or [B]: 1 = gradients written here, 0 = scene left to the dual-form kernel
  const int* only;            // nullptr or [B]: process only the scenes flagged non-zero (rescue pass after the dual form)
  unsigned flags;             // LCPB200_BWD_*: bit 0 = exact adjoint (transposed KKT system: K^T, W^T)
  const unsigned char* sload; // nullptr or [B][P.sbytes]: structure saved by the forward of the SAME inputs (skips the scan of Q, G, F)
  EngineSoA<T> soa;           // engine path: gradients w.r.t. the contact list instead of dense ones
  T *dmass, *dinertia, *dv, *dfext, *dnormal, *dp1, *dp2, *dmu, *drest;   // engine path outputs (any may be nullptr)
  long long* prof;
};

// ------------------------------------------------------------------ structure save / reuse
// The backward of a scene needs the same structure as its forward (components of F, block forms of G and F,
// column lists): 19 KB at cfg 3 against the 0.4 MB of dense Q, G, F it would have to scan again. The forward
// writes it to a per-scene slot of the handle's buffer, the backward of the same inputs reads it back.
__device__ __forceinline__ void copy16(unsigned char* dst, const unsigned char* src, int bytes) {
  const uint4* s4 = reinterpret_cast<const uint4*>(src);
  uint4* d4 = reinterpret_cast<uint4*>(dst);
  for (int i = threadIdx.x; i < (bytes >> 4); i += NT) d4[i] = s4[i];
}

__device__ __forceinline__ void save_structure(const CPlan& P, const Struct& st, bool ok, unsigned char* dst) {
  if (threadIdx.x == 0) *reinterpret_cast<int4*>(dst) = make_int4(ok ? st.ncomp : -1, st.cs, st.sh, st.m);
  if (!ok) return;
  const int c1 = P.o_x - P.o_Fd, c2 = P.o_y - P.o_qd, c3 = P.o_misc - P.o_rows;
  copy16(dst + 16, cnd_smem + P.o_Fd, c1);
  copy16(dst + 16 + c1, cnd_smem + P.o_qd, c2);
  copy16(dst + 16 + c1 + c2, cnd_smem + P.o_rows, c3);
}

// returns false when the forward found no structure for this scene (it went to the dual-form kernel)
__device__ __forceinline__ bool load_structure(const CPlan& P, Struct& st, const unsigned char* src) {
  const int4 hd = *reinterpret_cast<const int4*>(src);
  st.ncomp = hd.x; st.cs = hd.y; st.sh = hd.z; st.m = hd.w;
  if (hd.x < 0) return false;
  const int c1 = P.o_x - P.o_Fd, c2 = P.o_y - P.o_qd, c3 = P.o_misc - P.o_rows;
  copy16(cnd_smem + P.o_Fd, src + 16, c1);
  copy16(cnd_smem + P.o_qd, src + 16 + c1, c2);
  copy16(cnd_smem + P.o_rows, src + 16 + c1 + c2, c3);
  return true;
}

// ------------------------------------------------------------------ forward (pdipm.py:49-179), one scene
// Residuals of the current iterate (:82-96) into rx, rz, ry; returns s.z and the residual norm of :92-96.
template <typename T>
struct SzResid { T sz, resid; };

template <typename T, int CS>
__device__ __noinline__ SzResid<T> fwd_residuals(const CFwdArgs<T>& a, CSmem<T> S, Struct st, int sc) {
  const int nc_ = st.ncomp;                       // positions are slot-major: pos(c, r) = r * ncomp + c
  const CPlan& P = a.P;
  const int n = P.n, m = st.m, e = P.e, tid = threadIdx.x, pcap = P.pcap;      // m: this scene's rows (<= P.m, the stride)
  const T* p = a.p + (size_t)sc * n;
  const T* h = a.h + (size_t)sc * P.m;
  const T* b = e > 0 ? a.b + (size_t)sc * e : nullptr;
  for (int c = tid; c < n; c += NT) {                            // rx = G^T z + Q x + p (+ A^T y)
    T acc = 0;
    const int cnt = S.clcnt()[c];
    for (int l = 0; l < cnt; ++l) {
      const int cp = S.clist()[l * n + c], cc = cp >> 3, pp = cp & 7;
#pragma unroll
      for (int r = 0; r < CS; ++r) {
        const int i = S.rows()[r * nc_ + cc];
        if (i != 0xFFFF) acc = fma(S.Gd()[(size_t)pp * pcap + r * nc_ + cc], S.z()[i], acc);
      }
    }
    for (int k = 0; k < e; ++k) acc = fma(S.As()[k * n + c], S.y()[k], acc);
    S.rx()[c] = acc + S.qd()[c] * S.x()[c] + p[c];
  }
  for (int tt = tid; tt < (CS << st.sh); tt += NT) {              // rz = G x + s - h - F z
    const int r = tt >> st.sh, c = tt & ((1 << st.sh) - 1);
    if (c >= nc_) continue;
    const int pz = r * nc_ + c;
    const int i = S.rows()[pz];
    if (i == 0xFFFF) continue;
    const int nc = S.ncols()[c];
    T acc = 0;
    for (int q = 0; q < nc; ++q) acc = fma(S.Gd()[(size_t)q * pcap + pz], S.x()[S.ccols()[q * pcap + c]], acc);
    T fz = 0;
#pragma unroll
    for (int q = 0; q < CS; ++q) {
      const int j = S.rows()[q * nc_ + c];
      if (j != 0xFFFF) fz = fma(S.Fd()[(size_t)(r * CS + q) * nc_ + c], S.z()[j], fz);
    }
    S.rz()[i] = acc + S.s()[i] - h[i] - fz;
  }
  for (int k = tid; k < e; k += NT) {                            // ry = A x - b
    T acc = 0;
    for (int j = 0; j < n; ++j) acc = fma(S.As()[k * n + j], S.x()[j], acc);
    S.ry()[k] = acc - b[k];
  }
  __syncthreads();
  T q4[4] = {0, 0, 0, 0};                                        // s.z, |rz|^2, |ry|^2, |rx|^2
  for (int i = tid; i < m; i += NT) { q4[0] += S.s()[i] * S.z()[i]; q4[1] += S.rz()[i] * S.rz()[i]; }
  for (int i = tid; i < e; i += NT) q4[2] += S.ry()[i] * S.ry()[i];
  for (int i = tid; i < n; i += NT) q4[3] += S.rx()[i] * S.rx()[i];
  block_reduce<T, 4>(q4, OpSum(), T(0), S.red());
  const T sz = q4[0];
  const T mu = fabs(sz / T(m));                                  // :91
  return {sz, (e > 0 ? sqrt(q4[2]) : T(0)) + sqrt(q4[1]) + sqrt(q4[3]) + T(m) * mu};   // :92-96
}

// the best iterate so far becomes the output (:107-136)
template <typename T>
__device__ __noinline__ void fwd_store_best(const CFwdArgs<T>& a, CSmem<T> S, int m, int sc) {
  const CPlan& P = a.P;
  const int n = P.n, e = P.e, tid = threadIdx.x;
  for (int i = tid; i < n; i += NT) a.zhat[(size_t)sc * n + i] = S.x()[i];
  for (int i = tid; i < m; i += NT) { a.lam[(size_t)sc * P.m + i] = S.z()[i]; a.slack[(size_t)sc * P.m + i] = S.s()[i]; }
  for (int i = tid; i < e; i += NT) a.nu[(size_t)sc * e + i] = S.y()[i];
}

// affine step length and centering (:140-158): rs2 = (-mu sigma + ds dz) / s, the corrector's rs
template <typename T>
__device__ __noinline__ void fwd_centering(CSmem<T> S, int m, T mu, T sz) {
  const int tid = threadIdx.x;
  T stz, sts;
  get_steps(S.z(), S.dz(), S.s(), S.ds(), m, S.red(), stz, sts);
  const T alpha_aff = nan_min(nan_min(stz, sts), T(1));          // :142-144
  T t3[1] = {0};
  for (int i = tid; i < m; i += NT) t3[0] += (S.s()[i] + alpha_aff * S.ds()[i]) * (S.z()[i] + alpha_aff * S.dz()[i]);
  block_reduce<T, 1>(t3, OpSum(), T(0), S.red());
  const T ratio = t3[0] / sz;                                    // :146-150
  const T sig = ratio * ratio * ratio;
  const T musig = -mu * sig;                                     // :152-158
  for (int i = tid; i < m; i += NT) S.rs2()[i] = (musig + S.ds()[i] * S.dz()[i]) / S.s()[i];
  __syncthreads();
}

// affine + corrector direction and the step along it (:160-174); the corrector is in rx, rz (ds), rs2 (dz), ry
template <typename T>
__device__ __noinline__ void fwd_step(const CPlan& P, CSmem<T> S, int m) {
  const int n = P.n, e = P.e, tid = threadIdx.x;
  for (int i = tid; i < n; i += NT) S.dx()[i] += S.rx()[i];          // :160-163
  for (int i = tid; i < m; i += NT) { S.ds()[i] += S.rz()[i]; S.dz()[i] += S.rs2()[i]; }
  for (int i = tid; i < e; i += NT) S.dy()[i] += S.ry()[i];
  __syncthreads();
  T stz, sts;
  get_steps(S.z(), S.dz(), S.s(), S.ds(), m, S.red(), stz, sts);
  const T alpha = nan_min(T(0.999) * nan_min(stz, sts), T(1));   // :164-166
  for (int i = tid; i < n; i += NT) S.x()[i] += alpha * S.dx()[i];   // :171-174
  for (int i = tid; i < m; i += NT) { S.s()[i] += alpha * S.ds()[i]; S.z()[i] += alpha * S.dz()[i]; }
  for (int i = tid; i < e; i += NT) S.y()[i] += alpha * S.dy()[i];
  __syncthreads();
}

template <typename T, int NS, int CS, typename PF>
__device__ __forceinline__ void forward_scene(const CFwdArgs<T>& a, CSmem<T>& S, const Struct& st, PF& pf, int sc) {
  const CPlan& P = a.P;
  const int m = st.m;                                            // this scene's rows (<= P.m, the stride)
  {
    const int n = P.n, e = P.e, tid = threadIdx.x;
    const T* h = a.h + (size_t)sc * P.m;
    const T* b = e > 0 ? a.b + (size_t)sc * e : nullptr;
    // ---- initial point: d = 1, rhs (p, 0, -h, -b)                 :58-63
    for (int i = tid; i < m; i += NT) { S.d()[i] = T(1); S.rs2()[i] = T(0); S.rz()[i] = -h[i]; }
    for (int i = tid; i < n; i += NT) S.rx()[i] = a.p[(size_t)sc * n + i];
    for (int i = tid; i < e; i += NT) S.ry()[i] = -b[i];
    __syncthreads();
  }
  factor_kkt<T, NS, CS>(P, S, st, pf);
  solve_kkt<T, CS, NS>(P, S, st, pf, S.rx(), S.rs2(), S.rz(), P.e > 0 ? S.ry() : nullptr, S.x(), S.s(), S.z(), S.y());
  pf.count(CPH_FACTORS);
  pf.count(CPH_SOLVES);
  if (m == 0) {
    // engine path, a scene without contacts: no complementarity, the equality-constrained solve above is the
    // answer (engines.py:35-49 solves [[M, -Je^T], [Je, 0]] x = [M v + dt f; 0] directly in that case)
    fwd_store_best<T>(a, S, 0, sc);
    if (threadIdx.x == 0) { a.status[sc] = 2; a.iters[sc] = 0; if (a.resid) a.resid[sc] = T(0); }
    return;
  }
  {   // shift s and z to >= 1 where the row minimum is <= 0       :65-75
    const int tid = threadIdx.x;
    T mn[2] = {INFINITY, INFINITY};
    for (int i = tid; i < m; i += NT) { mn[0] = nan_min(mn[0], S.s()[i]); mn[1] = nan_min(mn[1], S.z()[i]); }
    block_reduce<T, 2>(mn, OpMin(), (T)INFINITY, S.red());
    for (int i = tid; i < m; i += NT) {
      if (mn[0] <= T(0)) S.s()[i] -= mn[0] - T(1);
      if (mn[1] <= T(0)) S.z()[i] -= mn[1] - T(1);
    }
    __syncthreads();
  }

  T best = nan("");
  bool have_best = false;
  int not_improved = 0, status = 0, it = 0;
  for (it = 0; it < a.max_iter; ++it) {
    const SzResid<T> r = fwd_residuals<T, CS>(a, S, st, sc);
    pf.lap(CPH_RESID);
    const T mu = fabs(r.sz / T(m));                                // :91

    // ---- best iterate / termination (per scene)                 :107-136
    // (the reference refactors before this test, :98-102; the factors of a terminating iteration
    // are never used, so the test comes first here)
    bool improved;
    if (!have_best) { improved = true; have_best = true; not_improved = 0; }
    else { improved = r.resid < best; not_improved = improved ? 0 : not_improved + 1; }
    if (improved) {
      best = r.resid;
      fwd_store_best<T>(a, S, m, sc);
    }
    if (not_improved == a.not_improved_lim) { status = 1; ++it; break; }
    if (best < a.eps) { status = 2; ++it; break; }
    if (mu > T(1e100)) { status = 3; ++it; break; }
    // the step below would make an iterate no residual is formed for: it can never become `best`, so the last
    // iteration ends here (status 0, iters == max_iter, as if it had run)
    if (it + 1 == a.max_iter) { ++it; break; }

    for (int i = threadIdx.x; i < m; i += NT) S.d()[i] = S.z()[i] / S.s()[i];     // :98
    __syncthreads();
    factor_kkt<T, NS, CS>(P, S, st, pf);                               // :100

    // ---- affine direction                                       :138-139   (rs = z)
    solve_kkt<T, CS, NS>(P, S, st, pf, S.rx(), S.z(), S.rz(), P.e > 0 ? S.ry() : nullptr, S.dx(), S.ds(), S.dz(), S.dy());
    fwd_centering<T>(S, m, mu, r.sz);
    pf.lap(CPH_STEP);
    // corrector: outputs land in rx / rz / ry (dead until the next residual phase)
    solve_kkt<T, CS, NS>(P, S, st, pf, nullptr, S.rs2(), nullptr, nullptr, S.rx(), S.rz(), S.rs2(), S.ry());
    // NOTE: ds_c -> S.rz(), dz_c -> S.rs2() (solve_kkt reads rs before it writes dz/ds of the same row)
    fwd_step<T>(P, S, m);
    pf.lap(CPH_STEP);
    pf.count(CPH_FACTORS);
    pf.count(CPH_SOLVES, 2);
  }
  if (threadIdx.x == 0) { a.status[sc] = status; a.iters[sc] = it; if (a.resid) a.resid[sc] = best; }
}

template <typename T, int NS, bool PROF>
__global__ void __launch_bounds__(NT, (NS <= 6) ? 2 : 1) cond_forward_kernel(const __grid_constant__ CFwdArgs<T> a) {
  const CPlan& P = a.P;
  CSmem<T> S(P);
  const int n = P.n, m = P.m, e = P.e, tid = threadIdx.x;
  __shared__ int singular_s;
  const T NANV = nan("");
  Prof<PROF> pf(PROF ? a.prof + (size_t)blockIdx.x * CPH_COUNT : nullptr);
  for (int sc = blockIdx.x; sc < a.B; sc += gridDim.x) {
    if (tid == 0) singular_s = 0;
    __syncthreads();
    pf.start();
    Struct st;
    const bool ok = a.soa.mass
        ? build_structure_soa<T>(P, S, st, a.soa, sc, e > 0 ? a.A + (size_t)sc * e * n : nullptr, &singular_s)
        : build_structure<T>(P, S, st, a.Q + (size_t)sc * n * n, a.G + (size_t)sc * m * n,
                             e > 0 ? a.A + (size_t)sc * e * n : nullptr, a.F + (size_t)sc * m * m, &singular_s);
    __syncthreads();
    if (a.ssave) save_structure(P, st, ok, a.ssave + (size_t)sc * P.sbytes);
    pf.lap(CPH_STRUCT);
    if (!ok) {
      if (singular_s) {                 // pdipm.py:361-368: the caller raises
        for (int i = tid; i < n; i += NT) a.zhat[(size_t)sc * n + i] = NANV;
        for (int i = tid; i < m; i += NT) { a.lam[(size_t)sc * m + i] = NANV; a.slack[(size_t)sc * m + i] = NANV; }
        for (int i = tid; i < e; i += NT) a.nu[(size_t)sc * e + i] = NANV;
        if (tid == 0) { a.status[sc] = -1; a.iters[sc] = 0; if (a.resid) a.resid[sc] = NANV; }
      } else if (tid == 0) {
        a.status[sc] = STATUS_UNSUPPORTED;     // the dual form (dense API) overwrites both; the engine path returns them
        a.iters[sc] = 0;
      }
      __syncthreads();
      continue;
    }
    if constexpr (LU_BW < NS - 1) mark_band_lu<T>(P, S, st);
    switch (st.cs) {
      case 1: forward_scene<T, NS, 1>(a, S, st, pf, sc); break;
      case 2: forward_scene<T, NS, 2>(a, S, st, pf, sc); break;
      case 3: forward_scene<T, NS, 3>(a, S, st, pf, sc); break;
      case 4: forward_scene<T, NS, 4>(a, S, st, pf, sc); break;
      case 5: forward_scene<T, NS, 5>(a, S, st, pf, sc); break;
      default: forward_scene<T, NS, 6>(a, S, st, pf, sc); break;
    }
    __syncthreads();
  }
}

// o[i][j] = f(i, j), row-major rows x cols, written by the whole CTA. When a row is a multiple of 16 bytes and o is
// 16-byte aligned a thread produces V = 16 / sizeof(T) consecutive elements of one row and stores them at once
// (the scalar form spent 26 % of the backward kernel's instructions on index bookkeeping and 4-byte stores).
template <typename T, typename F>
__device__ __forceinline__ void write_outer(T* __restrict__ o, int rows, int cols, F f) {
  constexpr int V = 16 / (int)sizeof(T);
  const int tid = threadIdx.x;
  if (cols % V == 0 && (reinterpret_cast<size_t>(o) & 15) == 0) {
    const int cv = cols / V, total = rows * cv;
    const int di = NT / cv, dj = NT - di * cv;
    int i = tid / cv, jv = tid - i * cv;
    for (int t = tid; t < total; t += NT) {
      const int j = jv * V;
      if (V == 4) {
        float4 w;
        w.x = (float)f(i, j); w.y = (float)f(i, j + 1); w.z = (float)f(i, j + 2); w.w = (float)f(i, j + 3);
        reinterpret_cast<float4*>(o)[t] = w;
      } else {
        double2 w;
        w.x = (double)f(i, j); w.y = (double)f(i, j + 1);
        reinterpret_cast<double2*>(o)[t] = w;
      }
      i += di; jv += dj;
      if (jv >= cv) { jv -= cv; ++i; }
    }
  } else {
    int i = tid / cols, j = tid - i * cols;
    const int di = NT / cols, dj = NT - di * cols;
    for (size_t t = tid; t < (size_t)rows * cols; t += NT) {
      o[t] = f(i, j);
      i += di; j += dj;
      if (j >= cols) { j -= cols; ++i; }
    }
  }
}

// ------------------------------------------------------------------ backward (lcp.py:37-64), one scene
// The gradients of one cotangent from the solve's dx, dlam, dnu: inputs of scene sc, outputs at row so.
template <typename T, int CS, typename PF>
__device__ __forceinline__ void backward_grads(const CBwdArgs<T>& a, CSmem<T>& S, const Struct& st, PF& pf, int sc, int so) {
  const CPlan& P = a.P;
  const int n = P.n, m = st.m, e = P.e, tid = threadIdx.x;
  const T* dx = S.dx(); const T* dlam = S.dz(); const T* dnu = S.dy();
  if (a.soa.mass) {
    // Engine path: the chain rule through the assembly (world.py:144-234, engines.py:50-116) applied to the
    // FACTORED gradients of lcp.py:52-63 -- dG = dlam (x) zhat + lam (x) dx, dF = -dlam (x) lam, dh = -dlam,
    // dQ = sym(dx (x) zhat), dp = dx -- evaluated only at the entries the assembly writes.
    const EngineSoA<T>& E = a.soa;
    const int nc = st.ncomp, nb = E.nb, ncs = E.nc;             // nc: this scene's contacts, ncs: array stride
    const int32_t* tb1 = E.b1 + (E.nc_s ? (size_t)sc * ncs : 0);
    const int32_t* tb2 = E.b2 + (E.nc_s ? (size_t)sc * ncs : 0);
    const T* v = E.v + (size_t)sc * n;
    const T* zh_ = S.x(); const T* lm = S.z();
    for (int c = tid; c < ncs; c += NT) {
      const size_t ic = (size_t)sc * ncs + c, oc = (size_t)so * ncs + c;
      if (c >= nc) {                                              // unused slots of a scene with fewer contacts
        if (a.dnormal) { a.dnormal[oc * 2] = 0; a.dnormal[oc * 2 + 1] = 0; }
        if (a.dp1) { a.dp1[oc * 2] = 0; a.dp1[oc * 2 + 1] = 0; }
        if (a.dp2) { a.dp2[oc * 2] = 0; a.dp2[oc * 2 + 1] = 0; }
        if (a.drest) a.drest[oc] = 0;
        if (a.dmu) a.dmu[oc] = 0;
        continue;
      }
      const T nx = E.normal[ic * 2], ny = E.normal[ic * 2 + 1];
      const T p1x = E.p1[ic * 2], p1y = E.p1[ic * 2 + 1], p2x = E.p2[ic * 2], p2y = E.p2[ic * 2 + 1];
      const bool two = tb2[c] < nb;                               // else body2 is a static obstacle: no columns
      const int j1 = 3 * tb1[c], j2 = two ? 3 * tb2[c] : j1;
      const T rc = E.rest[ic];
      const T dhc = -dlam[c] * (E.mode == 0 ? T(1) : T(1));      // dh = -dlam  (:55)
      T gnx = 0, gny = 0, g1x = 0, g1y = 0, g2x = 0, g2y = 0, jcv = 0;
      const int nrows = E.mode == 0 ? 3 : 1;
      const int rows_[3] = {c, nc + 2 * c, nc + 2 * c + 1};
      const T dxs[3] = {nx, ny, -ny}, dys[3] = {ny, -nx, nx};
      for (int q = 0; q < nrows; ++q) {
        const T ddx_ = dxs[q], ddy_ = dys[q];
        const int i = rows_[q];
        T g[6];
        for (int t = 0; t < 3; ++t) {
          g[t] = dlam[i] * zh_[j1 + t] + lm[i] * dx[j1 + t];      // dG[i][j1+t]  (:53)
          g[3 + t] = two ? dlam[i] * zh_[j2 + t] + lm[i] * dx[j2 + t] : T(0);
        }
        if (q == 0) {
          const T row[6] = {p1x * ddy_ - p1y * ddx_, ddx_, ddy_, -(p2x * ddy_ - p2y * ddx_), -ddx_, -ddy_};
          for (int t = 0; t < 3; ++t) jcv += row[t] * v[j1 + t] + row[3 + t] * (two ? v[j2 + t] : T(0));
          const T hs_ = E.mode == 0 ? rc : (T(1) - rc);            // h_c = (Jc v) rest  |  (Jc v)(1 - rest)
          for (int t = 0; t < 3; ++t) { g[t] += dhc * hs_ * v[j1 + t]; g[3 + t] += dhc * hs_ * (two ? v[j2 + t] : T(0)); }
        }
        const T gdx = -p1y * g[0] + g[1] + p2y * g[3] - g[4];
        const T gdy = p1x * g[0] + g[2] - p2x * g[3] - g[5];
        g1x += ddy_ * g[0]; g1y += -ddx_ * g[0];
        g2x += -ddy_ * g[3]; g2y += ddx_ * g[3];
        if (q == 0) { gnx += gdx; gny += gdy; }
        else if (q == 1) { gny += gdx; gnx += -gdy; }               // dir1 = (ny, -nx)
        else { gny += -gdx; gnx += gdy; }                           // dir2 = (-ny, nx)
      }
      if (a.dnormal) { a.dnormal[oc * 2] = gnx; a.dnormal[oc * 2 + 1] = gny; }
      if (a.dp1) { a.dp1[oc * 2] = g1x; a.dp1[oc * 2 + 1] = g1y; }
      if (a.dp2) { a.dp2[oc * 2] = g2x; a.dp2[oc * 2 + 1] = g2y; }
      if (a.drest) a.drest[oc] = E.mode == 0 ? dhc * jcv : -dhc * jcv;
      if (a.dmu) a.dmu[oc] = E.mode == 0 ? -(dlam[3 * nc + c] * lm[c]) : T(0);     // dF[gamma_c][c]  (:54)
    }
    for (int j = tid; j < n; j += NT) {
      const int body = j / 3, comp = j - 3 * body;
      const T md = comp == 0 ? E.inertia[(size_t)sc * nb + body] : E.mass[(size_t)sc * nb + body];
      const T dpj = E.mode == 0 ? dx[j] : T(0);                     // dp = dx (:52); post-stabilisation has p = 0
      if (a.dfext) a.dfext[(size_t)so * n + j] = E.dt * dpj;
      if (a.dv) {
        T acc = md * dpj;
        const int cnt = S.clcnt()[j];
        for (int l = 0; l < cnt; ++l) {                             // the contacts that touch this dof
          const int cp = S.clist()[l * n + j], c = cp >> 3, pslot = cp & 7;
          const T hs_ = E.mode == 0 ? E.rest[(size_t)sc * ncs + c] : (T(1) - E.rest[(size_t)sc * ncs + c]);
          acc += -dlam[c] * hs_ * S.Gd()[(size_t)pslot * P.pcap + c];      // dh_c d(h_c)/dv_j, Jc row = slot-0 rows of Gd
        }
        a.dv[(size_t)so * n + j] = acc;
      }
      const T dqjj = dx[j] * zh_[j];                                // dQ_jj = 1/2 (dx_j z_j + z_j dx_j)  (:61)
      if (comp == 0 && a.dinertia) a.dinertia[(size_t)so * nb + body] = dqjj + dpj * v[j];
    }
    __syncthreads();
    for (int body = tid; body < nb; body += NT) {
      if (!a.dmass) break;
      T acc = 0;
      for (int comp = 1; comp < 3; ++comp) {
        const int j = 3 * body + comp;
        acc += dx[j] * zh_[j] + (E.mode == 0 ? dx[j] : T(0)) * v[j];
      }
      a.dmass[(size_t)so * nb + body] = acc;
    }
    if (a.db && e > 0) for (int i = tid; i < e; i += NT) a.db[(size_t)so * e + i] = -dnu[i];
    if (a.dA && e > 0) {
      T* o = a.dA + (size_t)so * e * n;
      for (int i = 0; i < e; ++i)
        for (int j = tid; j < n; j += NT) o[(size_t)i * n + j] = dnu[i] * S.x()[j] + S.y()[i] * dx[j];
    }
    if (tid == 0 && a.done) a.done[sc] = 1;
    __syncthreads();
    pf.lap(CPH_GRADS);
    return;
  }
  if (a.dp) for (int i = tid; i < n; i += NT) a.dp[(size_t)so * n + i] = dx[i];                       // :52
  if (a.dh) for (int i = tid; i < m; i += NT) a.dh[(size_t)so * m + i] = -dlam[i];                    // :55
  if (a.db && e > 0) for (int i = tid; i < e; i += NT) a.db[(size_t)so * e + i] = -dnu[i];            // :58
  // the four dense outer products (0.4 MB per scene at cfg 3): 16-byte stores, V elements of one row per thread
  if (a.dG)                                                      // :53  dlam (x) zhat + lam (x) dx
    write_outer<T>(a.dG + (size_t)so * m * n, m, n, [&](int i, int j) { return dlam[i] * S.x()[j] + S.z()[i] * dx[j]; });
  if (a.dF)                                                      // :54  -dlam (x) lam
    write_outer<T>(a.dF + (size_t)so * m * m, m, m, [&](int i, int j) { return -(dlam[i] * S.z()[j]); });
  if (a.dA && e > 0)                                             // :57
    write_outer<T>(a.dA + (size_t)so * e * n, e, n, [&](int i, int j) { return dnu[i] * S.x()[j] + S.y()[i] * dx[j]; });
  if (a.dQ)                                                      // :61
    write_outer<T>(a.dQ + (size_t)so * n * n, n, n, [&](int i, int j) { return T(0.5) * (dx[i] * S.x()[j] + S.x()[i] * dx[j]); });
  if (tid == 0 && a.done) a.done[sc] = 1;
  __syncthreads();
  pf.lap(CPH_GRADS);
}

// One factorisation at the saved solution, then one solve and chain rule per cotangent r in [r0, r1): the
// factors, W and the structure in shared memory are read-only to solve_kkt, so every round sees the same matrix.
template <typename T, int NS, int CS, typename PF>
__device__ __forceinline__ void backward_scene(const CBwdArgs<T>& a, CSmem<T>& S, const Struct& st, PF& pf, int sc,
                                               int r0, int r1) {
  const CPlan& P = a.P;
  const int n = P.n, m = st.m, e = P.e, tid = threadIdx.x;
  const T* zh = a.zhat + (size_t)sc * n;
  const T* lam = a.lam + (size_t)sc * P.m;
  const T* slk = a.slack + (size_t)sc * P.m;
  const T* nu = e > 0 ? a.nu + (size_t)sc * e : nullptr;
  for (int i = tid; i < n; i += NT) S.x()[i] = zh[i];
  for (int i = tid; i < m; i += NT) {
    T d = lam[i] / slk[i];                                                              // :44
    // fp64 only: at the round-off floor (lambda, s ~ 1e-16) d spans 1e+-16 and the condensed matrix
    // K = Q + G^T (F + 1/d)^-1 G, which inherits the large entries, can no longer be factored (kappa u >= 1,
    // exact zero pivots). Clamping d to [1e-10, 1e10] moves the KKT diagonal of rows that are converged
    // to 1e-16 by < 1e-10 -- far below the 1e-4 at which the reference's own gradients are reproducible
    // there (tests/test_oracle.py) -- and keeps kappa(K) u <= 1e-6.
    if (sizeof(T) == 8) d = d > T(1e10) ? T(1e10) : (d < T(1e-10) ? T(1e-10) : d);
    S.z()[i] = lam[i]; S.s()[i] = slk[i]; S.d()[i] = d;
  }
  for (int i = tid; i < e; i += NT) S.y()[i] = nu[i];
  __syncthreads();
  const bool exact = (a.flags & 1u) != 0;
  factor_kkt<T, NS, CS>(P, S, st, pf, exact);                                               // :46  (m == 0: K = [[Q, A^T], [A, 0]])
  for (int r = r0; r < r1; ++r) {
    const int so = r * a.B + sc;                                  // output row of (cotangent r, scene sc)
    for (int i = tid; i < n; i += NT) S.rx()[i] = a.g[(size_t)so * n + i];
    for (int i = tid; i < m; i += NT) S.rs2()[i] = T(0);
    __syncthreads();
    solve_kkt<T, CS, NS>(P, S, st, pf, S.rx(), S.rs2(), nullptr, nullptr, S.dx(), S.ds(), S.dz(), S.dy(), exact);   // :47-50
    backward_grads<T, CS>(a, S, st, pf, sc, so);
  }
}

template <typename T, int NS, bool PROF>
__global__ void __launch_bounds__(NT, (NS <= 6) ? 2 : 1) cond_backward_kernel(const __grid_constant__ CBwdArgs<T> a) {
  const CPlan& P = a.P;
  CSmem<T> S(P);
  const int n = P.n, m = P.m, e = P.e, tid = threadIdx.x;
  __shared__ int singular_s;
  Prof<PROF> pf(PROF ? a.prof + (size_t)blockIdx.x * CPH_COUNT : nullptr);
  for (int w = blockIdx.x; w < a.B * a.chunks; w += gridDim.x) {
    const int sc = w / a.chunks, k = w - sc * a.chunks;
    if (a.only && !a.only[sc]) continue;
    if (tid == 0) singular_s = 0;
    __syncthreads();
    pf.start();
    Struct st;
    const bool ok = a.soa.mass
        ? build_structure_soa<T>(P, S, st, a.soa, sc, e > 0 ? a.A + (size_t)sc * e * n : nullptr, &singular_s)
        : a.sload
              ? load_structure(P, st, a.sload + (size_t)sc * P.sbytes)       // the forward of the same inputs found it
              : build_structure<T>(P, S, st, a.Q + (size_t)sc * n * n, a.G + (size_t)sc * m * n,
                                   e > 0 ? a.A + (size_t)sc * e * n : nullptr, a.F + (size_t)sc * m * m, &singular_s);
    __syncthreads();
    pf.lap(CPH_STRUCT);
    if (!ok) {
      if (tid == 0 && a.done) a.done[sc] = 0;
      __syncthreads();
      continue;
    }
    if constexpr (LU_BW < NS - 1) mark_band_lu<T>(P, S, st);   // also after load_structure: the saved column lists give the same answer
    const int r0 = (int)((long long)a.R * k / a.chunks), r1 = (int)((long long)a.R * (k + 1) / a.chunks);
    switch (st.cs) {
      case 1: backward_scene<T, NS, 1>(a, S, st, pf, sc, r0, r1); break;
      case 2: backward_scene<T, NS, 2>(a, S, st, pf, sc, r0, r1); break;
      case 3: backward_scene<T, NS, 3>(a, S, st, pf, sc, r0, r1); break;
      case 4: backward_scene<T, NS, 4>(a, S, st, pf, sc, r0, r1); break;
      case 5: backward_scene<T, NS, 5>(a, S, st, pf, sc, r0, r1); break;
      default: backward_scene<T, NS, 6>(a, S, st, pf, sc, r0, r1); break;
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------ Jacobian-vector products, engine path
// Forward-mode derivative of the engine solve (DESIGN.md section 8). At the saved iterate (zhat, lam, slack, nu)
// with the backward's clamp of d = lam / slack, the PDIPM residuals (pdipm.py:82-90) linearised in the inputs give
//     K [dx; ds; dz; dy] = -(r_x, 0, r_z, r_y),
//     r_x = dQ zhat + dp + dG^T lam + dA^T nu,   r_z = dG zhat - dF lam - dh,   r_y = dA zhat - db,
// K the NON-transposed matrix the forward factors; the tangent of zhat is dx. d(Q, p, G, h, F) is the directional
// derivative of the assembly (build_structure_soa), evaluated per contact and per dof, never as a dense matrix.
// Every tangent is [R][B][...] like CBwdArgs' cotangents, nullptr = zero.
// Dense inputs (soa.mass == nullptr): the structure comes from Q, G, A, F (or sload) as in cond_backward_kernel and
// d(Q, p, G, h, F) are the dense tangents tQ ... tF.

// Tangents of the engine's contact list, each [R][B][...] like the inputs it moves, nullptr = zero.
template <typename T>
struct EngineTangents {
  const T *mass, *inertia, *v, *fext, *normal, *p1, *p2, *mu, *rest, *A, *b;
};

template <typename T>
struct CJvpArgs {
  CPlan P;
  int B, R, chunks;           // work items (scene, chunk of tangents), as CBwdArgs
  const T *Q, *G, *A, *F;
  const T *zhat, *nu, *lam, *slack;
  EngineSoA<T> soa;
  EngineTangents<T> t;        // t.A, t.b serve both paths
  const T *tQ, *tp, *tG, *th, *tF;   // dense path: [R][B][...] or nullptr
  int* done;                  // dense path, as CBwdArgs
  const int* only;
  const unsigned char* sload;
  T* dz;                      // [R][B][n]
  long long* prof;
};

// Tangent of contact_row along (dx, dy) when the points move by (tp1, tp2) and the direction by (tdx, tdy).
template <typename T>
__device__ __forceinline__ void contact_row_tangent(T p1x, T p1y, T p2x, T p2y, T dx, T dy, T t1x, T t1y, T t2x,
                                                    T t2y, T tdx, T tdy, T (&r1)[3], T (&r2)[3]) {
  r1[0] = t1x * dy + p1x * tdy - t1y * dx - p1y * tdx; r1[1] = tdx; r1[2] = tdy;
  r2[0] = -(t2x * dy + p2x * tdy - t2y * dx - p2y * tdx); r2[1] = -tdx; r2[2] = -tdy;
}

// Right-hand side (r_x, r_z, r_y) of the engine JVP for tangent slot so of scene sc (nc contacts), shared by the
// condensed and banded kernels. The layout L says where the two families keep things:
//   L.x(), L.z(), L.y(): the saved iterate zhat, lam, nu;  L.rx(), L.rz(), L.ry(): where r_x, r_z, r_y go;
//   L.row(q, k): the slot of row q of contact k (0: normal, 1 and 2: friction, 3: the gamma row of mode 0);
//   L.walk(j, body, f): f(k, side) for every contact k touching dof j of `body`, side 1 when it is the contact's body2.
// One thread per contact and one per dof; the walk's order is the summation order of dG^T lam (deterministic).
template <typename T, typename L>
__device__ __forceinline__ void engine_jvp_rhs(const EngineSoA<T>& E, const EngineTangents<T>& t, L lay, int sc, int so,
                                            int n, int e, int nc) {
  const int tid = threadIdx.x, nb = E.nb, ncs = E.nc;
  const int32_t* tb1 = E.b1 + (E.nc_s ? (size_t)sc * ncs : 0);
  const int32_t* tb2 = E.b2 + (E.nc_s ? (size_t)sc * ncs : 0);
  const T* v = E.v + (size_t)sc * n;
  const T* tv = t.v ? t.v + (size_t)so * n : nullptr;
  const T* zh = lay.x(); const T* lm = lay.z();
  T* rz = lay.rz();
  auto tget = [](const T* p, size_t i) { return p ? p[i] : T(0); };
  // r_z, one thread per contact
  for (int k = tid; k < nc; k += NT) {
    const size_t ic = (size_t)sc * ncs + k, oc = (size_t)so * ncs + k;
    const int b1 = tb1[k], b2 = tb2[k];
    const bool two = b2 < nb;
    const T nx = E.normal[ic * 2], ny = E.normal[ic * 2 + 1];
    const T p1x = E.p1[ic * 2], p1y = E.p1[ic * 2 + 1], p2x = E.p2[ic * 2], p2y = E.p2[ic * 2 + 1];
    const T tnx = tget(t.normal, oc * 2), tny = tget(t.normal, oc * 2 + 1);
    const T t1x = tget(t.p1, oc * 2), t1y = tget(t.p1, oc * 2 + 1);
    const T t2x = tget(t.p2, oc * 2), t2y = tget(t.p2, oc * 2 + 1);
    T r1[3], r2[3], d1[3], d2[3];
    contact_row<T>(p1x, p1y, p2x, p2y, nx, ny, r1, r2);
    contact_row_tangent<T>(p1x, p1y, p2x, p2y, nx, ny, t1x, t1y, t2x, t2y, tnx, tny, d1, d2);
    T jv = 0, tjv = 0, gz = 0;                    // Jc v, d(Jc v), dJc zhat
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      const int j1 = 3 * b1 + q;
      jv += r1[q] * v[j1];
      tjv += d1[q] * v[j1] + (tv ? r1[q] * tv[j1] : T(0));
      gz += d1[q] * zh[j1];
      if (two) {
        const int j2 = 3 * b2 + q;
        jv += r2[q] * v[j2];
        tjv += d2[q] * v[j2] + (tv ? r2[q] * tv[j2] : T(0));
        gz += d2[q] * zh[j2];
      }
    }
    const T rc = E.rest[ic], trc = tget(t.rest, oc);
    if (E.mode == 0) {
      rz[lay.row(0, k)] = gz - (trc * jv + rc * tjv);                 // h_c = (Jc v) rest
      contact_row_tangent<T>(p1x, p1y, p2x, p2y, ny, -nx, t1x, t1y, t2x, t2y, tny, -tnx, d1, d2);
      T fz = 0;                                                        // dJf zhat (row f2 = -row f1)
#pragma unroll
      for (int q = 0; q < 3; ++q) { fz += d1[q] * zh[3 * b1 + q]; if (two) fz += d2[q] * zh[3 * b2 + q]; }
      rz[lay.row(1, k)] = fz;
      rz[lay.row(2, k)] = -fz;
      rz[lay.row(3, k)] = -(tget(t.mu, oc) * lm[k]);                  // F[gamma_k][k] = mu_k
    } else {
      rz[lay.row(0, k)] = gz - (tjv * (T(1) - rc) - trc * jv);        // h_c = (Jc v)(1 - rest)
    }
  }
  // r_x, one thread per dof; dG^T lam is gathered through the contacts the layout's walk yields
  for (int j = tid; j < n; j += NT) {
    const int body = j / 3, comp = j - 3 * body;
    const T q = comp == 0 ? E.inertia[(size_t)sc * nb + body] : E.mass[(size_t)sc * nb + body];
    const T tq = comp == 0 ? tget(t.inertia, (size_t)so * nb + body) : tget(t.mass, (size_t)so * nb + body);
    T acc = tq * zh[j];
    if (E.mode == 0) acc += tq * v[j] + q * (tv ? tv[j] : T(0)) + E.dt * tget(t.fext, (size_t)so * n + j);
    lay.walk(j, body, [&](int k, int side) {
      const size_t ic = (size_t)sc * ncs + k, oc = (size_t)so * ncs + k;
      const T* pp = side ? E.p2 : E.p1;
      const T* tp = side ? t.p2 : t.p1;
      const T px = pp[ic * 2], py = pp[ic * 2 + 1], tpx = tget(tp, oc * 2), tpy = tget(tp, oc * 2 + 1);
      const T nx = E.normal[ic * 2], ny = E.normal[ic * 2 + 1];
      const T tnx = tget(t.normal, oc * 2), tny = tget(t.normal, oc * 2 + 1);
      // d(row entry) along direction (dx, dy): [p x d, d] of this body (negated for body2)
      auto drow = [&](T dx, T dy, T tdx, T tdy) {
        return comp == 0 ? tpx * dy + px * tdy - tpy * dx - py * tdx : (comp == 1 ? tdx : tdy);
      };
      T g = drow(nx, ny, tnx, tny) * lm[k];
      if (E.mode == 0) g += drow(ny, -nx, tny, -tnx) * (lm[lay.row(1, k)] - lm[lay.row(2, k)]);
      acc += side ? -g : g;
    });
    if (e > 0 && t.A) {
      const T* tA = t.A + (size_t)so * e * n;
      for (int i = 0; i < e; ++i) acc += tA[(size_t)i * n + j] * lay.y()[i];
    }
    lay.rx()[j] = acc;
  }
  for (int i = tid; i < e; i += NT) {
    T acc = -tget(t.b, (size_t)so * e + i);
    if (t.A) {
      const T* tA = t.A + (size_t)so * e * n + (size_t)i * n;
      for (int j = 0; j < n; ++j) acc += tA[j] * zh[j];
    }
    lay.ry()[i] = acc;
  }
  __syncthreads();
}

// engine_jvp_rhs' layout in the condensed kernel: rows {k, nc + 2k, nc + 2k + 1, 3nc + k} of contact k, and the
// dof's ascending contact list.
template <typename T>
struct CondRows {
  CSmem<T> S;
  int n, nc;
  const int32_t* b1;
  __device__ __forceinline__ T* x() const { return S.x(); }
  __device__ __forceinline__ T* z() const { return S.z(); }
  __device__ __forceinline__ T* y() const { return S.y(); }
  __device__ __forceinline__ T* rx() const { return S.rx(); }
  __device__ __forceinline__ T* rz() const { return S.rz(); }
  __device__ __forceinline__ T* ry() const { return S.ry(); }
  __device__ __forceinline__ int row(int q, int k) const { return q == 0 ? k : (q == 3 ? 3 * nc + k : nc + 2 * k + q - 1); }
  template <typename F>
  __device__ __forceinline__ void walk(int j, int body, F f) const {
    const int cnt = S.clcnt()[j];
    for (int l = 0; l < cnt; ++l) {
      const int k = S.clist()[l * n + j] >> 3;
      f(k, b1[k] == body ? 0 : 1);
    }
  }
};

// Right-hand side of tangent slot so for dense inputs (CJvpArgs::tQ ... tF): r_x by columns (thread j walks column j
// of tG and tA: coalesced, no atomics), r_z and r_y by rows.
template <typename T>
__device__ __noinline__ void jvp_rhs_dense(const CJvpArgs<T>& a, CSmem<T> S, Struct st, int sc, int so) {
  const CPlan& P = a.P;
  const int n = P.n, m = st.m, e = P.e, tid = threadIdx.x;
  const T* zh = S.x(); const T* lm = S.z(); const T* nu = S.y();
  const T* tQ = a.tQ ? a.tQ + (size_t)so * n * n : nullptr;
  const T* tG = a.tG ? a.tG + (size_t)so * m * n : nullptr;
  const T* tF = a.tF ? a.tF + (size_t)so * m * m : nullptr;
  const T* tA = (a.t.A && e > 0) ? a.t.A + (size_t)so * e * n : nullptr;
  for (int j = tid; j < n; j += NT) {
    T acc = a.tp ? a.tp[(size_t)so * n + j] : T(0);
    if (tQ) for (int i = 0; i < n; ++i) acc = fma(tQ[(size_t)j * n + i], zh[i], acc);
    if (tG) for (int i = 0; i < m; ++i) acc = fma(tG[(size_t)i * n + j], lm[i], acc);
    if (tA) for (int k = 0; k < e; ++k) acc = fma(tA[(size_t)k * n + j], nu[k], acc);
    S.rx()[j] = acc;
  }
  for (int i = tid; i < m; i += NT) {
    T acc = a.th ? -a.th[(size_t)so * m + i] : T(0);
    if (tG) for (int j = 0; j < n; ++j) acc = fma(tG[(size_t)i * n + j], zh[j], acc);
    if (tF) for (int k = 0; k < m; ++k) acc = fma(-tF[(size_t)i * m + k], lm[k], acc);
    S.rz()[i] = acc;
  }
  for (int k = tid; k < e; k += NT) {
    T acc = a.t.b ? -a.t.b[(size_t)so * e + k] : T(0);
    if (tA) for (int j = 0; j < n; ++j) acc = fma(tA[(size_t)k * n + j], zh[j], acc);
    S.ry()[k] = acc;
  }
  __syncthreads();
}

// engine_jvp_rhs in the condensed layout, kept out of line so that the JVP kernel's registers stay with the
// factorisation and the solves.
template <typename T>
__device__ __noinline__ void jvp_rhs(const CJvpArgs<T>& a, CSmem<T> S, Struct st, int sc, int so) {
  const EngineSoA<T>& E = a.soa;
  engine_jvp_rhs<T>(E, a.t, CondRows<T>{S, a.P.n, st.ncomp, E.b1 + (E.nc_s ? (size_t)sc * E.nc : 0)}, sc, so, a.P.n,
                    a.P.e, st.ncomp);
}

// One factorisation of K (not transposed) at the saved solution, then one right-hand side and one solve per
// tangent r in [r0, r1). The prologue repeats backward_scene's: as one shared helper it moved ptxas' register
// allocation of both kernels, and the backward ran measurably slower (DESIGN.md section 8).
template <typename T, int NS, int CS, bool DENSE, typename PF>
__device__ __forceinline__ void jvp_scene(const CJvpArgs<T>& a, CSmem<T>& S, const Struct& st, PF& pf, int sc,
                                          int r0, int r1) {
  const CPlan& P = a.P;
  const int n = P.n, m = st.m, e = P.e, tid = threadIdx.x;
  const T* zh = a.zhat + (size_t)sc * n;
  const T* lam = a.lam + (size_t)sc * P.m;
  const T* slk = a.slack + (size_t)sc * P.m;
  for (int i = tid; i < n; i += NT) S.x()[i] = zh[i];
  for (int i = tid; i < m; i += NT) {
    T d = lam[i] / slk[i];
    if (sizeof(T) == 8) d = d > T(1e10) ? T(1e10) : (d < T(1e-10) ? T(1e-10) : d);   // backward_scene's clamp
    S.z()[i] = lam[i]; S.s()[i] = slk[i]; S.d()[i] = d; S.rs2()[i] = T(0);
  }
  for (int i = tid; i < e; i += NT) S.y()[i] = a.nu[(size_t)sc * e + i];
  __syncthreads();
  factor_kkt<T, NS, CS>(P, S, st, pf, false);
  for (int r = r0; r < r1; ++r) {
    const int so = r * a.B + sc;
    if constexpr (DENSE) jvp_rhs_dense<T>(a, S, st, sc, so);
    else jvp_rhs<T>(a, S, st, sc, so);
    solve_kkt<T, CS, NS>(P, S, st, pf, S.rx(), S.rs2(), S.rz(), e > 0 ? S.ry() : nullptr, S.dx(), S.ds(), S.dz(),
                         S.dy());
    for (int i = tid; i < n; i += NT) a.dz[(size_t)so * n + i] = S.dx()[i];
    if (DENSE && tid == 0 && a.done) a.done[sc] = 1;
    __syncthreads();
    pf.lap(CPH_GRADS);
  }
}

// DENSE (soa.mass == nullptr): the dense branch, its own instantiation so that the engine's is compiled without it.
template <typename T, int NS, bool PROF, bool DENSE>
__global__ void __launch_bounds__(NT, (NS <= 6) ? 2 : 1) cond_jvp_kernel(const __grid_constant__ CJvpArgs<T> a) {
  const CPlan& P = a.P;
  CSmem<T> S(P);
  const int n = P.n, e = P.e, tid = threadIdx.x;
  __shared__ int singular_s;
  Prof<PROF> pf(PROF ? a.prof + (size_t)blockIdx.x * CPH_COUNT : nullptr);
  for (int w = blockIdx.x; w < a.B * a.chunks; w += gridDim.x) {
    const int sc = w / a.chunks, k = w - sc * a.chunks;
    const int r0 = (int)((long long)a.R * k / a.chunks), r1 = (int)((long long)a.R * (k + 1) / a.chunks);
    if (DENSE && a.only && !a.only[sc]) continue;
    if (tid == 0) singular_s = 0;
    __syncthreads();
    pf.start();
    Struct st;
    const bool ok = !DENSE
        ? build_structure_soa<T>(P, S, st, a.soa, sc, e > 0 ? a.A + (size_t)sc * e * n : nullptr, &singular_s)
        : a.sload
              ? load_structure(P, st, a.sload + (size_t)sc * P.sbytes)
              : build_structure<T>(P, S, st, a.Q + (size_t)sc * n * n, a.G + (size_t)sc * P.m * n,
                                   e > 0 ? a.A + (size_t)sc * e * n : nullptr, a.F + (size_t)sc * P.m * P.m, &singular_s);
    __syncthreads();
    pf.lap(CPH_STRUCT);
    if (!ok) {
      if (!DENSE) {                               // the forward reported it (status -100 / -1): zero tangents
        for (int r = r0; r < r1; ++r)
          for (int i = tid; i < n; i += NT) a.dz[((size_t)r * a.B + sc) * n + i] = T(0);
      } else if (tid == 0 && a.done) {
        a.done[sc] = 0;                           // dense: left to the dual-form kernel
      }
      __syncthreads();
      continue;
    }
    if constexpr (LU_BW < NS - 1) mark_band_lu<T>(P, S, st);
    if constexpr (!DENSE) {
      switch (st.cs) {
        case 1: jvp_scene<T, NS, 1, false>(a, S, st, pf, sc, r0, r1); break;
        default: jvp_scene<T, NS, 4, false>(a, S, st, pf, sc, r0, r1); break;   // the engine builds 1 (mode 1) or 4 rows
      }
    } else {
      switch (st.cs) {                            // dense scenes: any component size, as in cond_backward_kernel
        case 1: jvp_scene<T, NS, 1, true>(a, S, st, pf, sc, r0, r1); break;
        case 2: jvp_scene<T, NS, 2, true>(a, S, st, pf, sc, r0, r1); break;
        case 3: jvp_scene<T, NS, 3, true>(a, S, st, pf, sc, r0, r1); break;
        case 4: jvp_scene<T, NS, 4, true>(a, S, st, pf, sc, r0, r1); break;
        case 5: jvp_scene<T, NS, 5, true>(a, S, st, pf, sc, r0, r1); break;
        default: jvp_scene<T, NS, 6, true>(a, S, st, pf, sc, r0, r1); break;
      }
    }
    __syncthreads();
  }
}

}  // namespace cnd
}  // namespace lcpb200
