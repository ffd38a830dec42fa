// lcp_solver.cuh -- per-scene PDIPM forward / implicit-diff backward kernels (v2).
//
// Restates (H100-native, one CTA per scene, persistent grid):
//   pdipm.py:357-408 pre_factor_kkt, :414-454 factor_kkt, :325-354 solve_kkt,
//   :49-179 forward, :182-186 get_step, lcp.py:22-64 LCPFunction.forward/backward.
//
// Residency (Plan.mode): 0 = T (padded m x m) fully in shared memory; 1 = split (lcp_lu.cuh):
// L-shaped part in shared memory, U12 spilled to L2; 2 = T in an L2 workspace (huge problems).
// Vectors always live in shared memory; G and Q^{-1} join them when there is room.
#pragma once
#include "lcp_lu.cuh"

namespace lcpb200 {

struct Plan {
  int n, m, e;
  int mp;                     // m padded to a multiple of the LU block size
  int m1;                     // rows held in `main` (== mp unless split)
  int nt;                     // threads per CTA
  int grid;                   // resident CTAs
  int mode;                   // 0 smem, 1 split, 2 L2
  int ldT, ldL, ldG, ldQi;
  int stage_ld;               // leading dimension for staging G in T's region during pre-factor (0 = no)
  int prefetch;               // 1: prefetch R into T's region with cp.async (0 via LCPB200_NO_PREFETCH, debugging)
  int lds;                    // leading dimension of the diagonal-block staging tile
  int G_smem, Qi_smem;
  int off_T, off_L, off_G, off_Qi, off_vec;   // shared offsets, in elements
  int smem_bytes;
  long long ws_per_cta;       // workspace elements per CTA
  long long w_Qi, w_R, w_T, w_U12, w_X, w_XA, w_S11, w_V, w_W, w_Fell, w_Gell;
};

// phases for the optional cycle counters; the last two are counts of the factorisations and the solves
// (forward + backward substitution) the forward kernel executed
enum { PH_PREFACTOR = 0, PH_LOADT, PH_LU, PH_SOLVE, PH_RESID, PH_STEP, PH_LU_DIAG, PH_LU_PANEL, PH_LU_UPDATE,
       PH_LU_DIAGWAIT, PH_LU_SLOWDIAG, PH_LU_BLOCKS, PH_LU_AHEAD, PH_LU_WAIT, PH_FACTORS, PH_SOLVES, PH_COUNT };

template <typename T>
struct Vecs {
  T *x, *s, *z, *y, *d;
  T *rx, *rz, *ry;
  T *hz, *hy, *te;
  T *tn, *tn2;
  T *dxa, *dsa, *dza, *dya;
  T *dxc, *dsc, *dzc, *dyc;
  T *rs2;
  T *qinv;                    // n: 1/diag(Q) when Q is diagonal (SceneCtx::qdiag)
  T *lt;                      // nb*(nb+4)+nb: transposed copy of the current diagonal block's L (look-ahead)
  T *scratch;                 // max(4 nt, mp) elements
  T *red;                     // 128 elements
  int *perm;                  // mp ints
  T *stage;                   // 2 x (nb + 4): pivot-row broadcast buffer of the diagonal-block LU
  T *bcast;                   // 4 scalars handed from the residual team to the whole CTA
  T *rdiag;                   // mp reciprocals of the U diagonal
  int *iflag;                 // 4 ints: [0] = rows were interchanged in the current diagonal block
  __host__ __device__ long long carve(T* base, int n, int mp, int e, int nt, int nb, int lds) {
    long long o = 0;
#define LCPB200_TAKE(ptr, cnt) do { ptr = base + o; o += ((cnt) + 3) & ~3; } while (0)
    LCPB200_TAKE(x, n); LCPB200_TAKE(s, mp); LCPB200_TAKE(z, mp); LCPB200_TAKE(y, e); LCPB200_TAKE(d, mp);
    LCPB200_TAKE(rx, n); LCPB200_TAKE(rz, mp); LCPB200_TAKE(ry, e);
    LCPB200_TAKE(hz, mp); LCPB200_TAKE(hy, e); LCPB200_TAKE(te, e);
    LCPB200_TAKE(tn, n); LCPB200_TAKE(tn2, n);
    LCPB200_TAKE(dxa, n); LCPB200_TAKE(dsa, mp); LCPB200_TAKE(dza, mp); LCPB200_TAKE(dya, e);
    LCPB200_TAKE(dxc, n); LCPB200_TAKE(dsc, mp); LCPB200_TAKE(dzc, mp); LCPB200_TAKE(dyc, e);
    LCPB200_TAKE(rs2, mp); LCPB200_TAKE(qinv, n); LCPB200_TAKE(lt, nb * (nb + 4) + nb);
    LCPB200_TAKE(scratch, 4 * nt > mp ? 4 * nt : mp); LCPB200_TAKE(red, 128);
    { T* pp; LCPB200_TAKE(pp, mp); perm = reinterpret_cast<int*>(pp); }
    LCPB200_TAKE(stage, 2 * (nb + 4)); LCPB200_TAKE(bcast, 4); LCPB200_TAKE(rdiag, mp);
    (void)lds;
    { T* pp; LCPB200_TAKE(pp, 4); iflag = reinterpret_cast<int*>(pp); }
#undef LCPB200_TAKE
    return o;
  }
};

template <typename T, int MODE>
struct SceneCtx {
  int n, m, e, mp, nt, off_vec, lds;
  const T *Q, *G, *A, *F;     // this scene's inputs (G may point at the shared copy)
  int ldG;
  T *Qi; int ldQi;
  TView<T, MODE> tv;
  T *R, *X, *XA, *S11, *Vm, *W;
  bool Rsaved;                // R points at a matrix saved by the forward pass (read-only)
  bool qdiag;                 // Q is diagonal: Q^{-1} v is an element-wise product with Vecs::qinv
  bool t_prefetched;          // R is already on its way into T's shared region (prefetch_T)
  bool transF;                // backward, exact adjoint: R is formed with F^T (the transposed KKT system)
  bool f_ell;                 // F has <= 4 non-zeros in every row: F z uses the ELL copy (Fell_v / Fell_i)
  T* Fell_v; int* Fell_i;     // [4][m] values / column indices (L2 workspace)
  bool g_ell_built;           // build_g_ell already ran for this scene (inside prefactor, from the staged copy)
  bool g_ell;                 // G (L2-resident) has <= 8 non-zeros per row and <= 32 per column: GEMVs use ELL copies
  T* Gr_v; int* Gr_i;         // [8][m]  row form:    G x
  T* Gc_v; int* Gc_i;         // [32][n] column form: G^T w
  int stage_ld;               // > 0: G may be staged in T's shared region with this leading dimension
  const T* Gsrc;              // this scene's G in global memory
  int* lu_flag;
  long long* prof;            // nullptr or PH_COUNT counters (thread 0 only)
  long long t_last;
  // shared-memory vectors, rebuilt from the namespace-scope shared array so the pointers are
  // provably shared inside every (non-inlined) device function
  __device__ __forceinline__ Vecs<T> vecs() const {
    Vecs<T> v;
    v.carve(smem_base<T>() + off_vec, n, mp, e, nt, Blk<T>::NB, lds);
    return v;
  }
};

template <typename C>
__device__ __forceinline__ void prof_start(C& c) { if (c.prof && threadIdx.x == 0) c.t_last = clock64(); }
template <typename C>
__device__ __forceinline__ void prof_lap(C& c, int ph) {
  if (c.prof && threadIdx.x == 0) { const long long t = clock64(); c.prof[ph] += t - c.t_last; c.t_last = t; }
}
template <typename C>
__device__ __forceinline__ void prof_count(C& c, int ph, int k = 1) {
  if (c.prof && threadIdx.x == 0) c.prof[ph] += k;
}

// ------------------------------------------------------------------ vector GEMVs
// out[r] = epi(r, sum_j A[r*lda+j] x[j]): one warp per row, RB rows (and all their vectors) in
// flight per warp so that an L2-resident matrix is streamed with deep memory-level parallelism.
template <typename T, typename Epi>
__device__ __forceinline__ void gemv_rows_v(const T* __restrict__ A, int lda, int M, int N, const T* x, Epi epi,
                                            const Team& tm) {
  using V = typename VecOf<T>::type;
  constexpr int VC = VecOf<T>::VC;
  constexpr int RB = 8;
  const int lane = tm.tid & 31, warp = tm.tid >> 5, nw = tm.nt >> 5;
  const bool vec_ok = (N % VC == 0) && (lda % VC == 0) && ((reinterpret_cast<uintptr_t>(A) & 15) == 0);
  if (vec_ok) {
    for (int r0 = warp * RB; r0 < M; r0 += nw * RB) {
      T acc[RB];
#pragma unroll
      for (int q = 0; q < RB; ++q) acc[q] = 0;
      for (int j = lane * VC; j < N; j += 32 * VC) {
        V av[RB];
#pragma unroll
        for (int q = 0; q < RB; ++q) av[q] = *reinterpret_cast<const V*>(A + (size_t)min(r0 + q, M - 1) * lda + j);
        T xv[VC];
        vec_get<T>(*reinterpret_cast<const V*>(x + j), xv);
#pragma unroll
        for (int q = 0; q < RB; ++q) {
          T a_[VC];
          vec_get<T>(av[q], a_);
#pragma unroll
          for (int t = 0; t < VC; ++t) acc[q] = fma(a_[t], xv[t], acc[q]);
        }
      }
#pragma unroll
      for (int q = 0; q < RB; ++q) acc[q] = warp_reduce(acc[q], OpSum());
      if (lane == 0) {
#pragma unroll
        for (int q = 0; q < RB; ++q)
          if (r0 + q < M) epi(r0 + q, acc[q]);
      }
    }
    tm.sync();
  } else {
    gemv_rows(A, lda, M, N, x, epi, tm);
  }
}

template <typename T, typename Epi>
__device__ __forceinline__ void gemv_rows_v(const T* __restrict__ A, int lda, int M, int N, const T* x, Epi epi) {
  gemv_rows_v(A, lda, M, N, x, epi, Team::cta());
}

// out[j] = epi(j, sum_i A[i*lda+j] w[i]): a thread owns one column vector and a slice of the rows;
// slices are combined through `scratch` (>= 4*blockDim.x elements).
template <typename T, typename Epi>
__device__ __forceinline__ void gemv_cols_v(const T* __restrict__ A, int lda, int M, int N, const T* w, T* scratch,
                                            Epi epi, const Team& tm) {
  using V = typename VecOf<T>::type;
  constexpr int VC = VecOf<T>::VC;
  const int NT = tm.nt;
  const int njv = N / VC;
  const bool vec_ok = (N % VC == 0) && (lda % VC == 0) && ((reinterpret_cast<uintptr_t>(A) & 15) == 0) && njv <= NT;
  if (!vec_ok) { gemv_cols(A, lda, M, N, w, scratch, epi, tm); return; }
  const int njp = (njv + 31) & ~31;
  const int parts = NT / njp;
  const int part = tm.tid / njp, jv = tm.tid - part * njp;
  T acc[VC];
#pragma unroll
  for (int t = 0; t < VC; ++t) acc[t] = 0;
  if (part < parts && jv < njv) {
    const T* col = A + jv * VC;
#pragma unroll 8
    for (int i = part; i < M; i += parts) {
      T av[VC];
      vec_get<T>(*reinterpret_cast<const V*>(col + (size_t)i * lda), av);
      const T wi = w[i];
#pragma unroll
      for (int t = 0; t < VC; ++t) acc[t] = fma(av[t], wi, acc[t]);
    }
    *reinterpret_cast<V*>(scratch + ((size_t)part * njv + jv) * VC) = vec_make(acc);
  }
  tm.sync();
  for (int j = tm.tid; j < N; j += NT) {
    T t = 0;
    for (int q = 0; q < parts; ++q) t += scratch[(size_t)q * N + j];
    epi(j, t);
  }
  tm.sync();
}

template <typename T, typename Epi>
__device__ __forceinline__ void gemv_cols_v(const T* __restrict__ A, int lda, int M, int N, const T* w, T* scratch,
                                            Epi epi) {
  gemv_cols_v(A, lda, M, N, w, scratch, epi, Team::cta());
}

// ------------------------------------------------------------------ R = G diag(qi) G^T + F
// Fast path of pdipm.py:378 for a diagonal Q (every mass matrix world.py:57-61 builds). Gs: a
// row-major copy of G (ld = ldg == 4 mod 32 words when staged in shared memory). Thread tile 8x8:
// rows rb + g + 4r, columns cb + cg + 8c -- both operand loads are vectors along k from
// consecutive rows, conflict-free. R and F are the L2/HBM arrays [m,m].
template <typename T>
__device__ __forceinline__ void gram_diag(const T* __restrict__ Gs, int ldg, const T* qi, const T* __restrict__ F,
                                          T* __restrict__ R, int m, int n, bool transF = false) {
  using V = typename VecOf<T>::type;
  constexpr int VC = VecOf<T>::VC;
  constexpr int TR = 8, TC = 8;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int g = lane >> 3, cg = lane & 7;
  const int ntr = (m + 31) / 32, ntc = (m + 63) / 64;
  for (int wt = warp; wt < ntr * ntc; wt += nw) {
    const int tr_ = wt / ntc, tc_ = wt - tr_ * ntc;
    const int rb = tr_ * 32 + g, cb = tc_ * 64 + cg;
    const T* ap[TR];
    const T* bp[TC];
#pragma unroll
    for (int r = 0; r < TR; ++r) ap[r] = Gs + (size_t)min(rb + 4 * r, m - 1) * ldg;
#pragma unroll
    for (int c = 0; c < TC; ++c) bp[c] = Gs + (size_t)min(cb + 8 * c, m - 1) * ldg;
    T acc[TR][TC];
#pragma unroll
    for (int r = 0; r < TR; ++r)
#pragma unroll
      for (int c = 0; c < TC; ++c) acc[r][c] = 0;
    for (int kc = 0; kc < n; kc += VC) {
      T a[TR][VC], qv[VC];
      vec_get<T>(*reinterpret_cast<const V*>(qi + kc), qv);
#pragma unroll
      for (int r = 0; r < TR; ++r) {
        vec_get<T>(*reinterpret_cast<const V*>(ap[r] + kc), a[r]);
#pragma unroll
        for (int t = 0; t < VC; ++t) a[r][t] *= qv[t];
      }
#pragma unroll
      for (int c = 0; c < TC; ++c) {
        T b[VC];
        vec_get<T>(*reinterpret_cast<const V*>(bp[c] + kc), b);
#pragma unroll
        for (int r = 0; r < TR; ++r)
#pragma unroll
          for (int t = 0; t < VC; ++t) acc[r][c] = fma(a[r][t], b[t], acc[r][c]);
      }
    }
#pragma unroll
    for (int r = 0; r < TR; ++r) {
      const int i = rb + 4 * r;
      if (i >= m) continue;
#pragma unroll
      for (int c = 0; c < TC; ++c) {
        const int j = cb + 8 * c;
        if (j < m) R[(size_t)i * m + j] = (transF ? F[(size_t)j * m + i] : F[(size_t)i * m + j]) + acc[r][c];
      }
    }
  }
  __syncthreads();
}

// ------------------------------------------------------------------ sparse copy of F
// Every F the engine builds (engines.py:66-72: E, mu, -E^T blocks) has at most 3 non-zeros per row,
// but the API hands it over dense (m^2 = 256 KB at cfg 3) and the residual needs F z every iteration.
// One pass per scene compacts the rows into ELL form (4 slots per row, in the L2 workspace); if any
// row has more non-zeros the dense GEMV stays. Sums run over the same non-zero terms as the dense
// product (adding zeros is exact), only their order differs.
template <typename T, int MODE>
__device__ __noinline__ void build_f_ell(SceneCtx<T, MODE>& c) {
  constexpr int KF = 4, CH = 8;                     // CH x 32 columns of a row in flight per lane
  const int m = c.m, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int dense = 0;
  for (int r = warp; r < m; r += nw) {
    const T* row = c.F + (size_t)r * m;
    int cnt = 0;
    for (int j0 = 0; j0 < m; j0 += 32 * CH) {
      T v[CH];
#pragma unroll
      for (int q = 0; q < CH; ++q) { const int j = j0 + q * 32 + lane; v[q] = j < m ? row[j] : T(0); }
#pragma unroll
      for (int q = 0; q < CH; ++q) {
        const bool nz = v[q] != T(0);
        const unsigned mask = __ballot_sync(FULL, nz);
        const int pos = cnt + __popc(mask & ((1u << lane) - 1u));
        if (nz && pos < KF) { c.Fell_v[(size_t)pos * m + r] = v[q]; c.Fell_i[(size_t)pos * m + r] = j0 + q * 32 + lane; }
        cnt += __popc(mask);
      }
    }
    if (cnt > KF) dense = 1;
    if (lane >= cnt && lane < KF) { c.Fell_v[(size_t)lane * m + r] = T(0); c.Fell_i[(size_t)lane * m + r] = 0; }
  }
  dense = __syncthreads_or(dense);
  c.f_ell = !dense;
}

// ------------------------------------------------------------------ sparse copies of G
// Contact Jacobians touch two bodies: <= 6 non-zeros per row of G (world.py:166-212), and a body
// column collects its contacts' rows. When G does not fit in shared memory every G x / G^T w of the
// iteration (5 per iteration) streams the dense 96 KB from L2; the ELL copies (8 slots per row,
// 32 per column, built once per scene by ordered ballot scans -- deterministic) cut that to 16 KB.
// Rows / columns with more non-zeros keep the dense path.
template <typename T, int MODE>
__device__ __noinline__ void build_g_ell(SceneCtx<T, MODE>& c, const T* Gp, int ldg) {
  // Gp/ldg: where to scan G from -- the copy staged in shared memory by prefactor when there is one
  // (the column scan is strided), else the global matrix
  constexpr int KR = 8, KC = 32, CH = 4;
  const int m = c.m, n = c.n, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  c.g_ell_built = true;
  if (c.G != c.Gsrc) { c.g_ell = false; return; }          // G lives in shared memory: dense is fine
  int dense = 0;
  for (int r = warp; r < m; r += nw) {                     // rows
    const T* row = Gp + (size_t)r * ldg;
    int cnt = 0;
    for (int j0 = 0; j0 < n; j0 += 32 * CH) {
      T v[CH];
#pragma unroll
      for (int q = 0; q < CH; ++q) { const int j = j0 + q * 32 + lane; v[q] = j < n ? row[j] : T(0); }
#pragma unroll
      for (int q = 0; q < CH; ++q) {
        const bool nz = v[q] != T(0);
        const unsigned mask = __ballot_sync(FULL, nz);
        const int pos = cnt + __popc(mask & ((1u << lane) - 1u));
        if (nz && pos < KR) { c.Gr_v[(size_t)pos * m + r] = v[q]; c.Gr_i[(size_t)pos * m + r] = j0 + q * 32 + lane; }
        cnt += __popc(mask);
      }
    }
    if (cnt > KR) dense = 1;
    if (lane >= cnt && lane < KR) { c.Gr_v[(size_t)lane * m + r] = T(0); c.Gr_i[(size_t)lane * m + r] = 0; }
  }
  for (int j = warp; j < n; j += nw) {                     // columns
    const T* col = Gp + j;
    int cnt = 0;
    for (int i0 = 0; i0 < m; i0 += 32 * CH) {
      T v[CH];
#pragma unroll
      for (int q = 0; q < CH; ++q) { const int i = i0 + q * 32 + lane; v[q] = i < m ? col[(size_t)i * ldg] : T(0); }
#pragma unroll
      for (int q = 0; q < CH; ++q) {
        const bool nz = v[q] != T(0);
        const unsigned mask = __ballot_sync(FULL, nz);
        const int pos = cnt + __popc(mask & ((1u << lane) - 1u));
        if (nz && pos < KC) { c.Gc_v[(size_t)pos * n + j] = v[q]; c.Gc_i[(size_t)pos * n + j] = i0 + q * 32 + lane; }
        cnt += __popc(mask);
      }
    }
    if (cnt > KC) dense = 1;
    if (lane >= cnt) { c.Gc_v[(size_t)lane * n + j] = T(0); c.Gc_i[(size_t)lane * n + j] = 0; }
  }
  dense = __syncthreads_or(dense);
  c.g_ell = !dense;
}

// G x and G^T w through whichever form is active (same epilogue interface as the dense GEMVs)
template <typename T, int MODE, typename Epi>
__device__ __forceinline__ void gemv_G_rows(SceneCtx<T, MODE>& c, const T* x, Epi epi, const Team& tm) {
  if (c.g_ell) {
    const int m = c.m;
    for (int i = tm.tid; i < m; i += tm.nt) {
      T acc = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k) acc = fma(c.Gr_v[(size_t)k * m + i], x[c.Gr_i[(size_t)k * m + i]], acc);
      epi(i, acc);
    }
    tm.sync();
  } else {
    gemv_rows_v(c.G, c.ldG, c.m, c.n, x, epi, tm);
  }
}
template <typename T, int MODE, typename Epi>
__device__ __forceinline__ void gemv_G_cols(SceneCtx<T, MODE>& c, const T* w, T* scratch, Epi epi, const Team& tm) {
  if (c.g_ell) {
    const int n = c.n;
    for (int j = tm.tid; j < n; j += tm.nt) {
      T acc0 = 0, acc1 = 0;
#pragma unroll
      for (int k = 0; k < 32; k += 2) {
        acc0 = fma(c.Gc_v[(size_t)k * n + j], w[c.Gc_i[(size_t)k * n + j]], acc0);
        acc1 = fma(c.Gc_v[(size_t)(k + 1) * n + j], w[c.Gc_i[(size_t)(k + 1) * n + j]], acc1);
      }
      epi(j, acc0 + acc1);
    }
    tm.sync();
  } else {
    gemv_cols_v(c.G, c.ldG, c.m, c.n, w, scratch, epi, tm);
  }
}

// ------------------------------------------------------------------ pre_factor_kkt (pdipm.py:357-408)
template <typename T, int MODE>
__device__ __noinline__ bool prefactor(SceneCtx<T, MODE>& c, int* flag) {
  const int n = c.n, m = c.m, e = c.e, tid = threadIdx.x, NT = blockDim.x;
  Vecs<T> v = c.vecs();
  if (tid == 0) *flag = 0;
  if (!c.Rsaved) {
    // F is read once, at the very end of this phase (R = G Q^-1 G^T + F), straight from HBM: pull it
    // towards L2 now so that the epilogue does not wait on DRAM
    const char* fp = reinterpret_cast<const char*>(c.F);
    const size_t lines = ((size_t)m * m * sizeof(T) + 127) / 128;
    for (size_t l = tid; l < lines; l += NT) asm volatile("prefetch.global.L2 [%0];" ::"l"(fp + l * 128));
  }
  // Q^{-1} (:362 factors Q; we keep the inverse so later Q-solves are GEMVs). Diagonal Q -- every
  // mass matrix the engine builds (world.py:57-61) -- is inverted directly.
  int offdiag = 0;
  for (int t = tid; t < n * n; t += NT) { const int i = t / n, j = t - i * n; if (i != j && c.Q[t] != T(0)) offdiag = 1; }
  offdiag = __syncthreads_or(offdiag);
  c.qdiag = !offdiag;
  if (!offdiag) {
    for (int t = tid; t < n * n; t += NT) {
      const int i = t / n, j = t - i * n;
      T val = 0;
      if (i == j) { const T q = c.Q[t]; if (!(q != T(0) && isfinite((double)q))) *flag = 1; val = T(1) / q; }
      c.Qi[(size_t)i * c.ldQi + j] = val;
      if (i == j) v.qinv[i] = val;
    }
    __syncthreads();
  } else {
    for (int t = tid; t < n * n; t += NT) { const int i = t / n, j = t - i * n; c.Qi[(size_t)i * c.ldQi + j] = c.Q[t]; }
    __syncthreads();
    invert_inplace(c.Qi, c.ldQi, n, flag, v.scratch);
  }
  const bool singular = (*flag != 0);
  __syncthreads();
  if (singular) return false;
  constexpr int VC_ = VecOf<T>::VC;
  if (c.Rsaved) {
    // R was saved by the forward pass (backward only): nothing to form. The G copies are still the ones the
    // staged branch below builds, so that the gradients do not depend on whether R was saved.
    if (!offdiag && n % VC_ == 0 && MODE != 2 && c.stage_ld > 0) build_g_ell(c, c.Gsrc, n);
  } else if (!offdiag && n % VC_ == 0) {
    // R = G diag(1/q) G^T + F with G staged in the (still unused) shared-memory region of T
    T* qd = v.scratch;                                           // n <= scratch
    for (int i = tid; i < n; i += NT) qd[i] = c.Qi[(size_t)i * c.ldQi + i];
    const int ldgs = c.stage_ld;
    if (MODE != 2 && ldgs > 0) {
      T* Gs = c.tv.main();
      const int nv = n / VC_;
      using V_ = typename VecOf<T>::type;
      const bool gal = (reinterpret_cast<uintptr_t>(c.Gsrc) & 15) == 0;
      if (gal) {
#pragma unroll 4
        for (int t = tid; t < m * nv; t += NT) {
          const int i = t / nv, j = (t - i * nv) * VC_;
          *reinterpret_cast<V_*>(Gs + (size_t)i * ldgs + j) = *reinterpret_cast<const V_*>(c.Gsrc + (size_t)i * n + j);
        }
      } else {
        for (int t = tid; t < m * n; t += NT) { const int i = t / n, j = t - i * n; Gs[(size_t)i * ldgs + j] = c.Gsrc[t]; }
      }
      __syncthreads();
      gram_diag<T>(Gs, ldgs, qd, c.F, c.R, m, n, c.transF);
      build_g_ell(c, Gs, ldgs);                                  // while the staged copy is still there
    } else {
      __syncthreads();
      gram_diag<T>(c.G, c.ldG, qd, c.F, c.R, m, n, c.transF);
    }
  } else {
    // X = Q^{-1} G^T ; R = G X + F                                 :378-379
    gemm_tiled<T, true>(c.X, m, c.Qi, c.ldQi, c.G, c.ldG, n, m, n, T(1), T(0));
    for (int t = tid; t < m * m; t += NT) { const int i = t / m, j = t - i * m; c.R[t] = c.transF ? c.F[(size_t)j * m + i] : c.F[t]; }
    __syncthreads();
    gemm_tiled<T, false>(c.R, m, c.G, c.ldG, c.X, m, m, m, n, T(1), T(1));
  }
  if (e > 0) {
    gemm_tiled<T, true>(c.XA, e, c.Qi, c.ldQi, c.A, n, n, e, n, T(1), T(0));          // :383
    gemm_tiled<T, false>(c.S11, e, c.A, n, c.XA, e, e, e, n, T(1), T(0));              // :384
    gemm_tiled<T, false>(c.Vm, e, c.G, c.ldG, c.XA, e, m, e, n, T(1), T(0));           // :385
    invert_inplace(c.S11, e, e, flag, v.scratch);                                    // :387
    gemm_tiled<T, true>(c.W, m, c.S11, e, c.Vm, e, e, m, e, T(1), T(0));               // :395
    if (!c.Rsaved) gemm_tiled<T, false>(c.R, m, c.Vm, e, c.W, m, m, m, e, T(-1), T(1));   // :403
  }
  return true;
}

// ------------------------------------------------------------------ prefetch of R for the next factor_kkt
// Only the diagonal of T = R + diag(1/d) changes between iterations but the LU overwrites T, so R
// is re-read every iteration. Once the corrector solve is done the old factors are dead: the copy
// R -> T's shared region is issued there with cp.async and completes behind the step-length /
// residual phases; factor_kkt then only adds the diagonal.
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  const unsigned sa = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sa), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

template <typename T, int MODE>
__device__ __forceinline__ void prefetch_T(SceneCtx<T, MODE>& c) {
  constexpr int VC = VecOf<T>::VC;
  if (MODE == 2) return;
  const int m = c.m, m1 = c.tv.m1, mp = c.mp, tid = threadIdx.x, NT = blockDim.x;
  if ((m % VC) != 0 || (reinterpret_cast<uintptr_t>(c.R) & 15) != 0) return;
  T* const tmain = c.tv.main();
  T* const tlow = (MODE == 1) ? c.tv.low() : tmain;
  const int mv = m / VC;                          // vectors per row of R
  const int r1 = min(m1, m);
  for (int t = tid; t < r1 * mv; t += NT) {       // main rows [0, m1) x columns [0, m)
    const int i = t / mv, j = (t - i * mv) * VC;
    cp_async16(tmain + (size_t)i * c.tv.ld + j, c.R + (size_t)i * m + j);
  }
  if (MODE == 1) {                                // low rows [m1, m) x columns [0, m1)
    const int m1v = m1 / VC;
    for (int t = tid; t < (m - m1) * m1v; t += NT) {
      const int i = m1 + t / m1v, j = (t % m1v) * VC;
      cp_async16(tlow + (size_t)(i - m1) * c.tv.ldl + j, c.R + (size_t)i * m + j);
    }
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
  c.t_prefetched = true;
}

// ------------------------------------------------------------------ first diagonal block, early
// The first diagonal block of T has no look-ahead partner inside the LU (ncu: 8 % of all samples were
// the other 15 warps waiting for it), but it only needs R (prefetched) and d = z/s of its own rows,
// both known before the residuals are formed. So the chain warp factors it while the rest of the
// CTA (a Team with its own named barrier) computes the residuals. Same arithmetic as factor_kkt:
// d = z/s, T_ii = R_ii + 1/d.
template <typename T, int MODE>
__device__ __forceinline__ LuVec make_luvec(SceneCtx<T, MODE>& c) {
  Vecs<T> v = c.vecs();
  LuVec lv;
  lv.o_perm_i = (int)(v.perm - smem_int(0));
  lv.o_flag_i = (int)(v.iflag - smem_int(0));
  lv.o_rmaxs = (int)(v.red - smem_base<T>());
  lv.o_rdiag = (int)(v.rdiag - smem_base<T>());
  lv.o_stage = (int)(v.stage - smem_base<T>());
  lv.lds = c.lds;
  lv.o_lt = (int)(v.lt - smem_base<T>()); lv.ldlt = Blk<T>::NB + 4;
  return lv;
}

template <typename T, int MODE>
__device__ __noinline__ void early_first_block(SceneCtx<T, MODE>& c) {
  constexpr int NB = Blk<T>::NB;
  Vecs<T> v = c.vecs();
  const int lane = threadIdx.x & 31;
  T* const tmain = c.tv.main();
  if (lane < NB) {
    const T d = v.z[lane] / v.s[lane];
    tmain[(size_t)lane * c.tv.ld + lane] += T(1) / d;
  }
  __syncwarp();
  const LuVec lv = make_luvec(c);
  diag_lu_rot<T, MODE, NB>(c.tv.main_, c.tv.ld, lv.o_perm_i, lv.o_rdiag, lv.o_flag_i, lv.o_stage, lv.o_lt, lv.ldlt, 0);
  if (c.prof && lane == 0) { c.prof[11] += 1; if (*smem_int(lv.o_flag_i)) c.prof[10] += 1; }
}

// ------------------------------------------------------------------ factor_kkt (pdipm.py:414-454)
// T = R + diag(1/d) (:427-429), padded with an identity block, loaded into the view, then LU (:431).
template <typename T, int MODE>
__device__ __noinline__ void factor_kkt(SceneCtx<T, MODE>& c, bool first_block_done = false) {
  using V = typename VecOf<T>::type;
  constexpr int VC = VecOf<T>::VC;
  const int m = c.m, mp = c.mp, m1 = c.tv.m1, tid = threadIdx.x, NT = blockDim.x;
  Vecs<T> v = c.vecs();
  const T* d = v.d;
  T* dinv = v.scratch;                                            // mp elements
  T* const tmain = c.tv.main();
  T* const tlow = (MODE == 1) ? c.tv.low() : tmain;
  for (int i = tid; i < mp; i += NT) dinv[i] = i < m ? T(1) / d[i] : T(1);
  __syncthreads();
  const bool vec_ok = (m % VC == 0) && ((reinterpret_cast<uintptr_t>(c.R) & 15) == 0);
  if (c.t_prefetched) {
    // R is arriving by cp.async (prefetch_T): finish it, fill the padding, add the diagonal
    c.t_prefetched = false;
    if (!first_block_done) cp_async_wait_all();
    const int mv = mp / VC;
    if (mp != m) {
      T z[VC];
#pragma unroll
      for (int q = 0; q < VC; ++q) z[q] = 0;
      for (int t = tid; t < m1 * mv; t += NT) {
        const int i = t / mv, j = (t - i * mv) * VC;
        if (!(i < m && j < m)) *reinterpret_cast<V*>(tmain + (size_t)i * c.tv.ld + j) = vec_make(z);
      }
      const int m1v = m1 / VC;
      for (int t = tid; t < (mp - m1) * m1v; t += NT) {
        const int i = m1 + t / m1v, j = (t % m1v) * VC;
        if (!(i < m && j < m)) *reinterpret_cast<V*>(tlow + (size_t)(i - m1) * c.tv.ldl + j) = vec_make(z);
      }
    }
    __syncthreads();
    // (the first diagonal block got its diagonal -- and its factorisation -- early, see early_first_block)
    for (int i = (first_block_done ? Blk<T>::NB : 0) + tid; i < m1; i += NT) tmain[(size_t)i * c.tv.ld + i] += dinv[i];
  } else if (vec_ok) {
    const int mv = mp / VC;
    constexpr int UB = 8;                          // independent L2 loads in flight per thread
    // main rows [0,m1) x all columns
    const int tot1 = m1 * mv;
    for (int t0 = tid; t0 < tot1; t0 += NT * UB) {
      V val[UB];
#pragma unroll
      for (int u = 0; u < UB; ++u) {
        const int t = t0 + u * NT;
        const int i = t / mv, j = (t - i * mv) * VC;
        T z[VC];
#pragma unroll
        for (int q = 0; q < VC; ++q) z[q] = 0;
        val[u] = (t < tot1 && i < m && j < m) ? *reinterpret_cast<const V*>(c.R + (size_t)i * m + j) : vec_make(z);
      }
#pragma unroll
      for (int u = 0; u < UB; ++u) {
        const int t = t0 + u * NT;
        if (t >= tot1) continue;
        const int i = t / mv, j = (t - i * mv) * VC;
        T w[VC];
        vec_get<T>(val[u], w);
#pragma unroll
        for (int q = 0; q < VC; ++q)
          if (j + q == i) w[q] += dinv[i];
        *reinterpret_cast<V*>(tmain + (size_t)i * c.tv.ld + j) = vec_make(w);
      }
    }
    // low rows [m1,mp) x columns [0,m1)
    const int m1v = m1 / VC;
    const int tot2 = (mp - m1) * m1v;
    for (int t0 = tid; t0 < tot2; t0 += NT * UB) {
      V val[UB];
#pragma unroll
      for (int u = 0; u < UB; ++u) {
        const int t = t0 + u * NT;
        const int i = m1 + t / m1v, j = (t % m1v) * VC;
        T z[VC];
#pragma unroll
        for (int q = 0; q < VC; ++q) z[q] = 0;
        val[u] = (t < tot2 && i < m && j < m) ? *reinterpret_cast<const V*>(c.R + (size_t)i * m + j) : vec_make(z);
      }
#pragma unroll
      for (int u = 0; u < UB; ++u) {
        const int t = t0 + u * NT;
        if (t >= tot2) continue;
        const int i = m1 + t / m1v, j = (t % m1v) * VC;
        *reinterpret_cast<V*>(tlow + (size_t)(i - m1) * c.tv.ldl + j) = val[u];
      }
    }
  } else {
    for (int t = tid; t < m1 * mp; t += NT) {
      const int i = t / mp, j = t - i * mp;
      T val = (i < m && j < m) ? c.R[(size_t)i * m + j] : T(0);
      if (i == j) val += dinv[i];
      tmain[(size_t)i * c.tv.ld + j] = val;
    }
    for (int t = tid; t < (mp - m1) * m1; t += NT) {
      const int i = m1 + t / m1, j = t % m1;
      tlow[(size_t)(i - m1) * c.tv.ldl + j] = (i < m && j < m) ? c.R[(size_t)i * m + j] : T(0);
    }
  }
  __syncthreads();
  prof_lap(c, PH_LOADT);
  const LuVec lv = make_luvec(c);
  lu_factor_view<T, MODE>(c.tv, c.R + (size_t)m1 * m + m1, m, (int)(dinv - smem_base<T>()), m, lv, c.prof, first_block_done);
  prof_lap(c, PH_LU);
}

// ------------------------------------------------------------------ solve_kkt (pdipm.py:325-354)
// Vectors are passed as element offsets into the shared array (-1 == zero vector) so that the
// pointers formed here are provably shared.
template <typename T, int MODE>
__device__ __noinline__ void solve_kkt(SceneCtx<T, MODE>& c, int o_rx, int o_rs, int o_rz, int o_ry,
                                       int o_dx, int o_ds, int o_dz, int o_dy) {
  const int n = c.n, m = c.m, e = c.e, tid = threadIdx.x, NT = blockDim.x;
  Vecs<T> v = c.vecs();
  T* const sb = smem_base<T>();
  const T* d = v.d;
  const T* rx = o_rx >= 0 ? sb + o_rx : nullptr;
  const T* rs = sb + o_rs;
  const T* rz = o_rz >= 0 ? sb + o_rz : nullptr;
  const T* ry = o_ry >= 0 ? sb + o_ry : nullptr;
  T* dx = sb + o_dx; T* ds = sb + o_ds; T* dz = sb + o_dz; T* dy = sb + o_dy;
  T* t = v.tn;                                                   // Q^{-1} rx      :333
  if (rx) {
    if (c.qdiag) {
      for (int i = tid; i < n; i += NT) t[i] = v.qinv[i] * rx[i];
      __syncthreads();
    } else {
      gemv_rows_v(c.Qi, c.ldQi, n, n, rx, [&](int i, T a) { t[i] = a; });
    }
    gemv_G_rows(c, t, [&](int i, T a) { v.hz[i] = a + rs[i] / d[i] - (rz ? rz[i] : T(0)); }, Team::cta());   // :337-340
    if (e > 0) gemv_rows_v(c.A, n, e, n, t, [&](int i, T a) { v.hy[i] = a - (ry ? ry[i] : T(0)); });
  } else {
    for (int i = tid; i < m; i += NT) v.hz[i] = rs[i] / d[i] - (rz ? rz[i] : T(0));
    for (int i = tid; i < e; i += NT) v.hy[i] = -(ry ? ry[i] : T(0));
    __syncthreads();
  }
  if (e > 0) {                                                   // block elimination of the e x e block  :342
    gemv_rows_v(c.S11, e, e, e, v.hy, [&](int i, T a) { v.te[i] = a; });
    gemv_rows_v(c.Vm, e, m, e, v.te, [&](int i, T a) { v.hz[i] -= a; });
  }
  lu_solve_view<T, MODE>(c.tv, (int)(v.perm - smem_int(0)), (int)(v.hz - smem_base<T>()), (int)(v.scratch - smem_base<T>()));               // hz <- T^{-1}(..) = -w_z   (hz[m..mp) stays 0)
  if (e > 0) gemv_rows_v(c.W, m, e, m, v.hz, [&](int i, T a) { dy[i] = -(v.te[i] - a); });
  for (int i = tid; i < m; i += NT) {
    const T wz = -v.hz[i];
    dz[i] = wz;                                                  // :351
    ds[i] = (-rs[i] - wz) / d[i];                                // :347,350
  }
  __syncthreads();
  T* g1 = v.tn2;                                                 // :344-349
  gemv_G_cols(c, dz, v.scratch, [&](int j, T a) { g1[j] = -(rx ? rx[j] : T(0)) - a; }, Team::cta());
  if (e > 0) gemv_cols_v(c.A, n, e, n, dy, v.scratch, [&](int j, T a) { g1[j] -= a; });
  if (c.qdiag) {
    for (int i = tid; i < n; i += NT) dx[i] = v.qinv[i] * g1[i];
    __syncthreads();
  } else {
    gemv_rows_v(c.Qi, c.ldQi, n, n, g1, [&](int i, T a) { dx[i] = a; });
  }
}

// ------------------------------------------------------------------ get_step (pdipm.py:182-186), per scene
template <typename T>
__device__ void get_steps(const T* z, const T* dz, const T* s, const T* ds, int m, T* red, T& step_z, T& step_s) {
  const T NEG_INF = -INFINITY, POS_INF = INFINITY;
  T mx[2] = {NEG_INF, NEG_INF};
  for (int i = threadIdx.x; i < m; i += blockDim.x) {
    mx[0] = nan_max(mx[0], -z[i] / dz[i]);
    mx[1] = nan_max(mx[1], -s[i] / ds[i]);
  }
  block_reduce<T, 2>(mx, OpMax(), NEG_INF, red);
  const T fz = (mx[0] > T(1)) ? mx[0] : T(1);                   // python max(1.0, a.max()): NaN -> 1.0
  const T fs = (mx[1] > T(1)) ? mx[1] : T(1);
  T mn[2] = {POS_INF, POS_INF};
  for (int i = threadIdx.x; i < m; i += blockDim.x) {
    const T az = (dz[i] > T(0)) ? fz : (-z[i] / dz[i]);
    const T as = (ds[i] > T(0)) ? fs : (-s[i] / ds[i]);
    mn[0] = nan_min(mn[0], az);
    mn[1] = nan_min(mn[1], as);
  }
  block_reduce<T, 2>(mn, OpMin(), POS_INF, red);
  step_z = mn[0];
  step_s = mn[1];
}

template <typename T>
struct FwdArgs {
  Plan P;
  int B;
  const T *Q, *p, *G, *h, *A, *b, *F;
  T *zhat, *nu, *lam, *slack, *resid;
  int *status, *iters;
  T eps;
  int not_improved_lim, max_iter;
  T* ws;
  T* Rsave;                   // nullptr or [B,m,m]: R of every scene, for the backward pass
  long long* prof;            // nullptr or [grid][PH_COUNT]
  int fallback_only;          // 1: solve only the scenes the condensed kernel flagged (status == -100)
};

template <typename T, int MODE>
__device__ void setup_ctx(SceneCtx<T, MODE>& c, const Plan& P, T* sm, T* ws, int* lu_flag, long long* prof) {
  c.n = P.n; c.m = P.m; c.e = P.e; c.mp = P.mp; c.nt = P.nt; c.off_vec = P.off_vec; c.lds = P.lds;
  c.Qi = P.Qi_smem ? sm + P.off_Qi : ws + P.w_Qi; c.ldQi = P.ldQi;
  c.tv.mp = P.mp; c.tv.m1 = P.m1;
  c.tv.main_.off = P.off_T; c.tv.main_.g = ws + P.w_T; c.tv.low_.off = P.off_L; c.tv.low_.g = nullptr;
  c.tv.ld = P.ldT; c.tv.ldl = P.ldL;
  c.tv.u12 = ws + P.w_U12;
  c.R = ws + P.w_R; c.X = ws + P.w_X; c.XA = ws + P.w_XA; c.S11 = ws + P.w_S11;
  c.Vm = ws + P.w_V; c.W = ws + P.w_W;
  c.Fell_v = ws + P.w_Fell; c.Fell_i = reinterpret_cast<int*>(ws + P.w_Fell + (long long)4 * P.m); c.f_ell = false;
  c.Gr_v = ws + P.w_Gell; c.Gr_i = reinterpret_cast<int*>(ws + P.w_Gell + (long long)8 * P.m);
  c.Gc_v = ws + P.w_Gell + (long long)16 * P.m; c.Gc_i = reinterpret_cast<int*>(ws + P.w_Gell + (long long)16 * P.m + (long long)32 * P.n);
  c.g_ell = false; c.g_ell_built = false;
  c.Rsaved = false; c.transF = false; c.qdiag = false; c.t_prefetched = false; c.stage_ld = P.stage_ld; c.Gsrc = nullptr;
  c.lu_flag = lu_flag;
  c.prof = prof ? prof + (size_t)blockIdx.x * PH_COUNT : nullptr;
  Vecs<T> v = c.vecs();
  // padded tails: never written again
  for (int i = P.m + threadIdx.x; i < P.mp; i += blockDim.x) {
    v.hz[i] = 0; v.s[i] = 1; v.z[i] = 1; v.d[i] = 1; v.rz[i] = 0; v.rs2[i] = 0;
    v.dsa[i] = 0; v.dza[i] = 0; v.dsc[i] = 0; v.dzc[i] = 0;
  }
  __syncthreads();
}

template <typename T, int MODE>
__device__ void bind_scene(SceneCtx<T, MODE>& c, const Plan& P, T* sm, const T* Q, const T* G, const T* A, const T* F) {
  const int n = P.n, m = P.m;
  c.Q = Q; c.A = A; c.F = F; c.Gsrc = G; c.g_ell_built = false; c.g_ell = false; c.f_ell = false;
  {   // padded tails: a NaN produced by the previous scene must not leak into this one
    Vecs<T> v = c.vecs();
    for (int i = P.m + threadIdx.x; i < P.mp; i += blockDim.x) {
      v.hz[i] = 0; v.s[i] = 1; v.z[i] = 1; v.d[i] = 1; v.rz[i] = 0; v.rs2[i] = 0;
      v.dsa[i] = 0; v.dza[i] = 0; v.dsc[i] = 0; v.dzc[i] = 0;
    }
  }
  if (P.G_smem) {
    T* Gs = sm + P.off_G;
    for (int t = threadIdx.x; t < m * n; t += blockDim.x) { int i = t / n, j = t - i * n; Gs[(size_t)i * P.ldG + j] = G[t]; }
    c.G = Gs; c.ldG = P.ldG;
  } else {
    c.G = G; c.ldG = n;
  }
  __syncthreads();
}

// ------------------------------------------------------------------ forward (pdipm.py:49-179)
template <typename T, int MODE>
__global__ void __launch_bounds__(512, 1) lcp_forward_kernel(const FwdArgs<T> a) {
  T* sm = smem_base<T>();
  __shared__ int flag;
  __shared__ int lu_flag_s;
  const Plan& P = a.P;
  const int n = P.n, m = P.m, e = P.e, tid = threadIdx.x, NT = blockDim.x;
  SceneCtx<T, MODE> c;
  setup_ctx<T, MODE>(c, P, sm, a.ws + (size_t)blockIdx.x * P.ws_per_cta, &lu_flag_s, a.prof);
  Vecs<T> v = c.vecs();
  T* const sb = sm;
  auto off = [&](const T* p_) { return (int)(p_ - sb); };
  const T NANV = nan("");

  for (int sc = blockIdx.x; sc < a.B; sc += gridDim.x) {
    if (a.fallback_only && a.status[sc] != -100) continue;       // solved by lcp_condensed.cuh
    const T* p = a.p + (size_t)sc * n;
    const T* h = a.h + (size_t)sc * m;
    const T* b = e > 0 ? a.b + (size_t)sc * e : nullptr;
    T* o_x = a.zhat + (size_t)sc * n;
    T* o_z = a.lam + (size_t)sc * m;
    T* o_s = a.slack + (size_t)sc * m;
    T* o_y = e > 0 ? a.nu + (size_t)sc * e : nullptr;
    prof_start(c);
    bind_scene(c, P, sm, a.Q + (size_t)sc * n * n, a.G + (size_t)sc * m * n,
               e > 0 ? a.A + (size_t)sc * e * n : nullptr, a.F + (size_t)sc * m * m);
    if (a.Rsave) c.R = a.Rsave + (size_t)sc * m * m;      // form R directly in the saved buffer

    if (!prefactor(c, &flag)) {
      for (int i = tid; i < n; i += NT) o_x[i] = NANV;
      for (int i = tid; i < m; i += NT) { o_z[i] = NANV; o_s[i] = NANV; }
      for (int i = tid; i < e; i += NT) o_y[i] = NANV;
      if (tid == 0) { a.status[sc] = -1; a.iters[sc] = 0; if (a.resid) a.resid[sc] = NANV; }
      __syncthreads();
      continue;
    }
    build_f_ell(c);
    if (!c.g_ell_built) build_g_ell(c, c.Gsrc, n);
    prof_lap(c, PH_PREFACTOR);

    // ---- initial point: d = 1, rhs (p, 0, -h, -b)                 :58-63
    for (int i = tid; i < m; i += NT) { v.d[i] = T(1); v.rs2[i] = T(0); v.rz[i] = -h[i]; }
    for (int i = tid; i < n; i += NT) v.rx[i] = p[i];
    for (int i = tid; i < e; i += NT) v.ry[i] = -b[i];
    __syncthreads();
    factor_kkt(c);
    solve_kkt(c, off(v.rx), off(v.rs2), off(v.rz), e > 0 ? off(v.ry) : -1, off(v.x), off(v.s), off(v.z), off(v.y));
    prof_count(c, PH_FACTORS);
    prof_count(c, PH_SOLVES);
    {   // shift s and z to >= 1 where the row minimum is <= 0       :65-75
      T mn[2] = {INFINITY, INFINITY};
      for (int i = tid; i < m; i += NT) { mn[0] = nan_min(mn[0], v.s[i]); mn[1] = nan_min(mn[1], v.z[i]); }
      block_reduce<T, 2>(mn, OpMin(), (T)INFINITY, v.red);
      for (int i = tid; i < m; i += NT) {
        if (mn[0] <= T(0)) v.s[i] -= mn[0] - T(1);
        if (mn[1] <= T(0)) v.z[i] -= mn[1] - T(1);
      }
      __syncthreads();
    }
    prof_lap(c, PH_SOLVE);

    T best = NANV;
    bool have_best = false;
    int not_improved = 0, status = 0, it = 0;
    for (it = 0; it < a.max_iter; ++it) {
      // ---- residuals                                              :82-96
      // When R has been prefetched into T (every iteration but the first) the chain warp factors the
      // first diagonal block now (early_first_block) and the other warps form the residuals as a Team.
      const bool overlap = c.t_prefetched && MODE != 2 && c.mp == m && NT >= 128;
      Team tm = Team::cta();
      bool in_team = true;
      if (overlap) {
        cp_async_wait_all();
        __syncthreads();                                           // every thread's part of R has landed
        tm.tid = tid; tm.nt = NT - 32; tm.bar = 3;
        in_team = tid < NT - 32;
        if (!in_team) early_first_block(c);
      }
      if (in_team) {
        const int TN = tm.nt;
        gemv_G_cols(c, v.z, v.scratch, [&](int j, T acc) { v.rx[j] = acc; }, tm);
        if (e > 0) gemv_cols_v(c.A, n, e, n, v.y, v.scratch, [&](int j, T acc) { v.rx[j] = acc + v.rx[j]; }, tm);
        if (c.qdiag) {
          for (int i = tid; i < n; i += TN) v.rx[i] = v.rx[i] + c.Q[(size_t)i * n + i] * v.x[i] + p[i];
          tm.sync();
        } else {
          gemv_rows_v(c.Q, n, n, n, v.x, [&](int i, T acc) { v.rx[i] = v.rx[i] + acc + p[i]; }, tm);
        }
        gemv_G_rows(c, v.x, [&](int i, T acc) { v.rz[i] = acc + v.s[i] - h[i]; }, tm);
        if (c.f_ell) {
          for (int i = tid; i < m; i += TN) {
            T acc = 0;
#pragma unroll
            for (int k = 0; k < 4; ++k) acc = fma(c.Fell_v[(size_t)k * m + i], v.z[c.Fell_i[(size_t)k * m + i]], acc);
            v.rz[i] -= acc;
          }
          tm.sync();
        } else {
          gemv_rows_v(c.F, m, m, m, v.z, [&](int i, T acc) { v.rz[i] -= acc; }, tm);
        }
        if (e > 0) gemv_rows_v(c.A, n, e, n, v.x, [&](int i, T acc) { v.ry[i] = acc - b[i]; }, tm);
        T q[4] = {0, 0, 0, 0};                                      // s.z, |rz|^2, |ry|^2, |rx|^2
        for (int i = tid; i < m; i += TN) { q[0] += v.s[i] * v.z[i]; q[1] += v.rz[i] * v.rz[i]; }
        for (int i = tid; i < e; i += TN) q[2] += v.ry[i] * v.ry[i];
        for (int i = tid; i < n; i += TN) q[3] += v.rx[i] * v.rx[i];
        block_reduce<T, 4>(q, OpSum(), T(0), v.red, tm);
        if (tid == 0) { v.bcast[0] = q[0]; v.bcast[1] = q[1]; v.bcast[2] = q[2]; v.bcast[3] = q[3]; }
        for (int i = tid; i < m; i += TN) v.d[i] = v.z[i] / v.s[i];     // :98
      }
      __syncthreads();
      const T sz = v.bcast[0];
      const T mu = fabs(sz / T(m));                               // :91
      const T resid = (e > 0 ? sqrt(v.bcast[2]) : T(0)) + sqrt(v.bcast[1]) + sqrt(v.bcast[3]) + T(m) * mu;   // :92-96
      prof_lap(c, PH_RESID);
      const bool last = it + 1 == a.max_iter;    // no step follows: its direction would make an unread iterate
      if (!last) { factor_kkt(c, overlap); prof_count(c, PH_FACTORS); }     // :100

      // ---- best iterate / termination (per scene)                 :107-136
      bool improved;
      if (!have_best) { improved = true; have_best = true; not_improved = 0; }
      else { improved = resid < best; not_improved = improved ? 0 : not_improved + 1; }
      if (improved) {
        best = resid;
        for (int i = tid; i < n; i += NT) o_x[i] = v.x[i];
        for (int i = tid; i < m; i += NT) { o_z[i] = v.z[i]; o_s[i] = v.s[i]; }
        for (int i = tid; i < e; i += NT) o_y[i] = v.y[i];
      }
      if (not_improved == a.not_improved_lim) { status = 1; ++it; break; }
      if (best < a.eps) { status = 2; ++it; break; }
      if (mu > T(1e100)) { status = 3; ++it; break; }
      if (last) { ++it; break; }

      // ---- affine direction                                       :138-139   (rs = z)
      solve_kkt(c, off(v.rx), off(v.z), off(v.rz), e > 0 ? off(v.ry) : -1, off(v.dxa), off(v.dsa), off(v.dza), off(v.dya));
      prof_lap(c, PH_SOLVE);
      T stz, sts;
      get_steps(v.z, v.dza, v.s, v.dsa, m, v.red, stz, sts);
      const T alpha_aff = nan_min(nan_min(stz, sts), T(1));       // :142-144
      T t3[1] = {0};
      for (int i = tid; i < m; i += NT) t3[0] += (v.s[i] + alpha_aff * v.dsa[i]) * (v.z[i] + alpha_aff * v.dza[i]);
      block_reduce<T, 1>(t3, OpSum(), T(0), v.red);
      const T ratio = t3[0] / sz;                                 // :146-150
      const T sig = ratio * ratio * ratio;
      const T musig = -mu * sig;                                  // :152-158
      for (int i = tid; i < m; i += NT) v.rs2[i] = (musig + v.dsa[i] * v.dza[i]) / v.s[i];
      __syncthreads();
      prof_lap(c, PH_STEP);
      solve_kkt(c, -1, off(v.rs2), -1, -1, off(v.dxc), off(v.dsc), off(v.dzc), off(v.dyc));
      // the factors are dead from here on. R goes to T for the last iteration too, although that one factors
      // nothing: the prefetch is what splits its residuals over a team (above), and the same split keeps the
      // last residual, and so `best`, bit for bit what a factoring iteration would compute
      if (it + 1 < a.max_iter && P.prefetch) prefetch_T(c);
      prof_lap(c, PH_SOLVE);
      for (int i = tid; i < n; i += NT) v.dxa[i] += v.dxc[i];    // :160-163
      for (int i = tid; i < m; i += NT) { v.dsa[i] += v.dsc[i]; v.dza[i] += v.dzc[i]; }
      for (int i = tid; i < e; i += NT) v.dya[i] += v.dyc[i];
      __syncthreads();
      get_steps(v.z, v.dza, v.s, v.dsa, m, v.red, stz, sts);
      const T alpha = nan_min(T(0.999) * nan_min(stz, sts), T(1));   // :164-166
      for (int i = tid; i < n; i += NT) v.x[i] += alpha * v.dxa[i];  // :171-174
      for (int i = tid; i < m; i += NT) { v.s[i] += alpha * v.dsa[i]; v.z[i] += alpha * v.dza[i]; }
      for (int i = tid; i < e; i += NT) v.y[i] += alpha * v.dya[i];
      __syncthreads();
      prof_lap(c, PH_STEP);
      prof_count(c, PH_SOLVES, 2);
    }
    // early exit or the last iteration (R prefetched, never factored): drain before T's region is reused
    if (c.t_prefetched) { cp_async_wait_all(); c.t_prefetched = false; }
    if (tid == 0) { a.status[sc] = status; a.iters[sc] = it; if (a.resid) a.resid[sc] = best; }
    __syncthreads();
  }
}

// ------------------------------------------------------------------ backward (lcp.py:37-64)
template <typename T>
struct BwdArgs {
  Plan P;
  int B;
  // R cotangents per scene: g and every gradient output are [R][B][...], slot r of scene sc at row r B + sc.
  // A work item is (scene, chunk): chunk k of `chunks` factors the scene's KKT matrix once and solves for the
  // cotangents [R k / chunks, R (k + 1) / chunks).
  int R, chunks;
  const T *Q, *G, *A, *F;
  const T *zhat, *nu, *lam, *slack, *g;
  T *dQ, *dp, *dG, *dh, *dA, *db, *dF;
  unsigned flags;
  T* ws;
  const T* Rsave;             // nullptr (recompute R) or the matrices saved by the forward pass
  long long* prof;
  const int* skip;            // nullptr or [B]: non-zero = gradients already written by lcp_condensed.cuh
  int* bad;                   // nullptr or [B], zeroed by the caller: set to 1 when a solve of the scene produced
                              // non-finite dx / dlam (LU broke down); the OR over its chunks and cotangents
};

// The saved iterate (zhat, lam, slack, nu) of scene sc into x, z, s, y, with d = lam / slack (:44, no clamp) and
// rs2 = 0; then K (transposed for the exact adjoint) is factored once for every right-hand side of the work item.
template <typename T, int MODE>
__device__ __forceinline__ void factor_saved(SceneCtx<T, MODE>& c, const Plan& P, T* sm, int* flag, int sc,
                                             const T* Q, const T* G, const T* A, const T* F, const T* zhat,
                                             const T* nu, const T* lam_, const T* slack, const T* Rsave, bool transF) {
  const int n = P.n, m = P.m, e = P.e, tid = threadIdx.x, NT = blockDim.x;
  Vecs<T> v = c.vecs();
  bind_scene(c, P, sm, Q + (size_t)sc * n * n, G + (size_t)sc * m * n, e > 0 ? A + (size_t)sc * e * n : nullptr,
             F + (size_t)sc * m * m);
  const T* zh = zhat + (size_t)sc * n;
  const T* lam = lam_ + (size_t)sc * m;
  const T* slk = slack + (size_t)sc * m;
  const T* nus = e > 0 ? nu + (size_t)sc * e : nullptr;
  c.transF = transF;                   // the saved R holds F, so it is not used for the transposed system
  if (Rsave && !c.transF) { c.R = const_cast<T*>(Rsave) + (size_t)sc * m * m; c.Rsaved = true; }
  prefactor(c, flag);                  // singular Q was already reported by the forward pass
  prof_lap(c, PH_PREFACTOR);
  for (int i = tid; i < n; i += NT) v.x[i] = zh[i];
  for (int i = tid; i < m; i += NT) { v.z[i] = lam[i]; v.s[i] = slk[i]; v.d[i] = lam[i] / slk[i]; v.rs2[i] = T(0); }   // :44
  for (int i = tid; i < e; i += NT) v.y[i] = nus[i];
  __syncthreads();
  factor_kkt(c);                                            // :46
}

// bad[sc] = 1 when the solve left a non-finite dx or dlam (the LU broke down); never cleared here.
template <typename T>
__device__ __forceinline__ void flag_nonfinite(int* bad, int sc, const T* dx, const T* dlam, int n, int m) {
  const int tid = threadIdx.x, NT = blockDim.x;
  int nf = 0;
  for (int i = tid; i < n; i += NT) nf |= !isfinite((double)dx[i]);
  for (int i = tid; i < m; i += NT) nf |= !isfinite((double)dlam[i]);
  nf = __syncthreads_or(nf);
  if (tid == 0 && nf) bad[sc] = 1;
}

template <typename T, int MODE>
__global__ void __launch_bounds__(512, 1) lcp_backward_kernel(const BwdArgs<T> a) {
  T* sm = smem_base<T>();
  __shared__ int flag;
  __shared__ int lu_flag_s;
  const Plan& P = a.P;
  const int n = P.n, m = P.m, e = P.e, tid = threadIdx.x, NT = blockDim.x;
  SceneCtx<T, MODE> c;
  setup_ctx<T, MODE>(c, P, sm, a.ws + (size_t)blockIdx.x * P.ws_per_cta, &lu_flag_s, a.prof);
  Vecs<T> v = c.vecs();
  T* const sb = sm;
  auto off = [&](const T* p_) { return (int)(p_ - sb); };

  for (int w = blockIdx.x; w < a.B * a.chunks; w += gridDim.x) {
    const int sc = w / a.chunks, k = w - sc * a.chunks;
    if (a.skip && a.skip[sc]) continue;
    prof_start(c);
    factor_saved(c, P, sm, &flag, sc, a.Q, a.G, a.A, a.F, a.zhat, a.nu, a.lam, a.slack, a.Rsave, (a.flags & 1u) != 0);
    const int r0 = (int)((long long)a.R * k / a.chunks), r1 = (int)((long long)a.R * (k + 1) / a.chunks);
    for (int r = r0; r < r1; ++r) {
      const size_t so = (size_t)r * a.B + sc;                   // output row of (cotangent r, scene sc)
      for (int i = tid; i < n; i += NT) v.rx[i] = a.g[so * n + i];
      __syncthreads();
      solve_kkt(c, off(v.rx), off(v.rs2), -1, -1, off(v.dxa), off(v.dsa), off(v.dza), off(v.dya));   // :47-50
      prof_lap(c, PH_SOLVE);
      const T* dx = v.dxa; const T* dlam = v.dza; const T* dnu = v.dya;
      if (a.bad) flag_nonfinite(a.bad, sc, dx, dlam, n, m);
      if (a.dp) for (int i = tid; i < n; i += NT) a.dp[so * n + i] = dx[i];                       // :52
      if (a.dh) for (int i = tid; i < m; i += NT) a.dh[so * m + i] = -dlam[i];                    // :55
      if (a.db && e > 0) for (int i = tid; i < e; i += NT) a.db[so * e + i] = -dnu[i];            // :58
      if (a.dG) {                                                    // :53  dlam (x) zhat + lam (x) dx
        T* o = a.dG + so * m * n;
        for (int t = tid; t < m * n; t += NT) { int i = t / n, j = t - i * n; o[t] = dlam[i] * v.x[j] + v.z[i] * dx[j]; }
      }
      if (a.dF) {                                                    // :54  -dlam (x) lam
        T* o = a.dF + so * m * m;
        for (int t = tid; t < m * m; t += NT) { int i = t / m, j = t - i * m; o[t] = -(dlam[i] * v.z[j]); }
      }
      if (a.dA && e > 0) {                                           // :57
        T* o = a.dA + so * e * n;
        for (int t = tid; t < e * n; t += NT) { int i = t / n, j = t - i * n; o[t] = dnu[i] * v.x[j] + v.y[i] * dx[j]; }
      }
      if (a.dQ) {                                                    // :61
        T* o = a.dQ + so * n * n;
        for (int t = tid; t < n * n; t += NT) { int i = t / n, j = t - i * n; o[t] = T(0.5) * (dx[i] * v.x[j] + v.x[i] * dx[j]); }
      }
      __syncthreads();
      prof_lap(c, PH_STEP);
    }
  }
}

// ------------------------------------------------------------------ Jacobian-vector products (dense inputs)
// Forward-mode derivative of the solve (DESIGN.md section 8, dense path). At the saved iterate, with d = lam / slack
// unclamped as in the backward, the PDIPM residuals (pdipm.py:82-90) linearised in the inputs give
//     K [dx; ds; dz; dy] = -(r_x, 0, r_z, r_y),
//     r_x = tQ zhat + tp + tG^T lam + tA^T nu,   r_z = tG zhat - tF lam - th,   r_y = tA zhat - tb,
// K the NON-transposed matrix the forward factors; the tangent of zhat is dx. Every tangent is [R][B][...] with the
// shape of its input, nullptr = zero; work items are (scene, chunk of tangents) as in BwdArgs.
template <typename T>
struct JvpArgs {
  Plan P;
  int B, R, chunks;
  const T *Q, *G, *A, *F;
  const T *zhat, *nu, *lam, *slack;
  const T *tQ, *tp, *tG, *th, *tA, *tb, *tF;
  T* dz;                      // [R][B][n]
  T* ws;
  const T* Rsave;
  long long* prof;
  const int* skip;            // as BwdArgs
  int* bad;
};

template <typename T, int MODE>
__global__ void __launch_bounds__(512, 1) lcp_jvp_kernel(const JvpArgs<T> a) {
  T* sm = smem_base<T>();
  __shared__ int flag;
  __shared__ int lu_flag_s;
  const Plan& P = a.P;
  const int n = P.n, m = P.m, e = P.e, tid = threadIdx.x, NT = blockDim.x;
  SceneCtx<T, MODE> c;
  setup_ctx<T, MODE>(c, P, sm, a.ws + (size_t)blockIdx.x * P.ws_per_cta, &lu_flag_s, a.prof);
  Vecs<T> v = c.vecs();
  T* const sb = sm;
  auto off = [&](const T* p_) { return (int)(p_ - sb); };

  for (int w = blockIdx.x; w < a.B * a.chunks; w += gridDim.x) {
    const int sc = w / a.chunks, k = w - sc * a.chunks;
    if (a.skip && a.skip[sc]) continue;
    prof_start(c);
    factor_saved(c, P, sm, &flag, sc, a.Q, a.G, a.A, a.F, a.zhat, a.nu, a.lam, a.slack, a.Rsave, false);
    const int r0 = (int)((long long)a.R * k / a.chunks), r1 = (int)((long long)a.R * (k + 1) / a.chunks);
    for (int r = r0; r < r1; ++r) {
      const size_t so = (size_t)r * a.B + sc;
      const T* tQ = a.tQ ? a.tQ + so * n * n : nullptr;
      const T* tG = a.tG ? a.tG + so * m * n : nullptr;
      const T* tF = a.tF ? a.tF + so * m * m : nullptr;
      const T* tA = (a.tA && e > 0) ? a.tA + so * e * n : nullptr;
      // row products first (one warp per row), then the column sums: thread j walks column j of tG and tA
      if (tQ) gemv_rows_v(tQ, n, n, n, v.x, [&](int i, T acc) { v.rx[i] = acc; });
      else { for (int i = tid; i < n; i += NT) v.rx[i] = T(0); }
      // r_z: each row is written by one GEMV epilogue at a time (gemv_rows_v syncs at its end, not at its start)
      if (tG) gemv_rows_v(tG, n, m, n, v.x, [&](int i, T acc) { v.rz[i] = acc; });
      if (tF) gemv_rows_v(tF, m, m, m, v.z, [&](int i, T acc) { v.rz[i] = (tG ? v.rz[i] : T(0)) - acc; });
      if (!tG && !tF) { for (int i = tid; i < m; i += NT) v.rz[i] = T(0); }
      if (tA) gemv_rows_v(tA, n, e, n, v.x, [&](int i, T acc) { v.ry[i] = acc; });
      else { for (int i = tid; i < e; i += NT) v.ry[i] = T(0); }
      __syncthreads();
      for (int j = tid; j < n; j += NT) {
        T acc = a.tp ? a.tp[so * n + j] : T(0);
        if (tG) for (int i = 0; i < m; ++i) acc = fma(tG[(size_t)i * n + j], v.z[i], acc);
        if (tA) for (int i = 0; i < e; ++i) acc = fma(tA[(size_t)i * n + j], v.y[i], acc);
        v.rx[j] += acc;
      }
      if (a.th) for (int i = tid; i < m; i += NT) v.rz[i] -= a.th[so * m + i];
      if (a.tb && e > 0) for (int i = tid; i < e; i += NT) v.ry[i] -= a.tb[so * e + i];
      __syncthreads();
      solve_kkt(c, off(v.rx), off(v.rs2), off(v.rz), e > 0 ? off(v.ry) : -1, off(v.dxa), off(v.dsa), off(v.dza), off(v.dya));
      prof_lap(c, PH_SOLVE);
      if (a.bad) flag_nonfinite(a.bad, sc, v.dxa, v.dza, n, m);
      for (int i = tid; i < n; i += NT) a.dz[so * n + i] = v.dxa[i];
      __syncthreads();
    }
  }
}

}  // namespace lcpb200
