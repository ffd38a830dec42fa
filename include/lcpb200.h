/* lcpb200.h -- C ABI of the H100-native batched LCP contact solver.
 *
 * The reference (locuslab/lcp-physics) is pure Python and has no FFI; this
 * header is the boundary a maintainer binds with ctypes (see INTEGRATION.md).
 * Every entry point replaces a reference interface on the hot path
 * (paths relative to the reference tree):
 *
 *   lcpb200_forward          lcp_physics/lcp/lcp.py:22-35   LCPFunction.forward
 *                            = lcp/solvers/pdipm.py:357-408 pre_factor_kkt
 *                            + lcp/solvers/pdipm.py:49-179  forward (PDIPM loop)
 *                            + pdipm.py:414-454 factor_kkt, :325-354 solve_kkt,
 *                              :182-186 get_step
 *   lcpb200_backward         lcp_physics/lcp/lcp.py:37-64   LCPFunction.backward
 *   lcpb200_assemble         lcp_physics/physics/world.py:144-234 (M,Jc,Jf,E,mu,
 *                            restitutions) + physics/engines.py:50-74 (G,F,h,p)
 *   lcpb200_assemble_backward  autograd through the same assembly
 *   lcpb200_forward_host / lcpb200_backward_host
 *                            the same calls with HOST buffers (pinned or
 *                            pageable); H2D/D2H copies are done inside, chunked
 *                            and overlapped with the kernels.
 *
 * Conventions
 *   - All matrices are dense, row-major, batch-major and contiguous, exactly
 *     the tensors LCPFunction receives: Q[B,n,n] p[B,n] G[B,m,n] h[B,m]
 *     A[B,e,n] b[B,e] F[B,m,m].  e == 0  <=>  A == b == NULL
 *     (the reference passes 1-D empty tensors, engines.py:59-60).
 *   - dtype: LCPB200_F32 or LCPB200_F64; all floating buffers share it.
 *   - Device pointers unless the function name ends in _host.
 *   - `stream` is a cudaStream_t passed as void*; NULL = legacy default stream.
 *   - Return value 0 = OK; non-zero = error, text via lcpb200_last_error_string().
 *     No exceptions cross the ABI.  Per-scene solver status is reported in
 *     `status[B]` (see LCPB200_STATUS_*): a singular Q sets
 *     LCPB200_STATUS_SINGULAR_Q and the caller raises the reference's
 *     RuntimeError (pdipm.py:361-368).
 *   - Scenes are independent: per-scene termination and per-scene get_step
 *     maximum (SURVEY.md F4: <= 1.5e-12 rel from the batch-coupled reference).
 *   - Two kernel families (DESIGN.md section 3). Scenes with the engine's structure (diagonal Q, sparse
 *     G, block-sparse F) are solved through the condensed n x n KKT system, formed / factored in fp64
 *     without pivoting (it is quasi-definite). Other scenes fall back, per scene, to the dual m x m
 *     form of the reference with threshold partial pivoting restricted to the LU's diagonal blocks
 *     (the reference pivots over whole columns on CPU tensors and not at all on CUDA tensors,
 *     pdipm.py:18 `pivot=not x.is_cuda`).
 *   - One stream at a time per handle (the handle owns the workspace).
 */
#ifndef LCPB200_H
#define LCPB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LCPB200_VERSION 200

#define LCPB200_F32 0
#define LCPB200_F64 1

/* per-scene status written by lcpb200_forward */
#define LCPB200_STATUS_MAX_ITER      0  /* ran all max_iter iterations            */
#define LCPB200_STATUS_NOT_IMPROVED  1  /* not_improved_lim non-improving iters   */
#define LCPB200_STATUS_CONVERGED     2  /* best residual < eps                    */
#define LCPB200_STATUS_DIVERGED      3  /* mu > 1e100                             */
#define LCPB200_STATUS_SINGULAR_Q   -1  /* zero / non-finite pivot factoring Q    */

/* flags for lcpb200_backward */
#define LCPB200_BWD_BUG_COMPATIBLE   0u /* reference behaviour: un-transposed KKT (SURVEY.md F6) */
#define LCPB200_BWD_EXACT_ADJOINT    1u /* transposed KKT system (true adjoint)                  */
#define LCPB200_BWD_REUSE_STRUCTURE  2u /* dense calls only: (Q, G, A, F) are the inputs of the
                                          * last lcpb200_forward on this handle (same B): reuse the
                                          * block structure it found instead of scanning the dense
                                          * matrices again (19 KB instead of 0.4 MB per scene at
                                          * config 3). Ignored when nothing matching was saved.    */

typedef struct lcpb200_handle_s* lcpb200_handle_t;

int         lcpb200_version(void);
const char* lcpb200_last_error_string(void);

/* Create a solver for problems of size (n, m, e) in `dtype` on CUDA device
 * `device`. The handle owns a small per-CTA workspace (independent of B). */
int lcpb200_create(int dtype, int n, int m, int e, int device, lcpb200_handle_t* out);
int lcpb200_destroy(lcpb200_handle_t h);
size_t lcpb200_workspace_bytes(lcpb200_handle_t h);
/* Describe the launch plan (threads, dynamic smem, grid, which matrices are
 * smem-resident) into `buf` -- for logs and DESIGN.md. */
int lcpb200_describe(lcpb200_handle_t h, char* buf, size_t len);

/* Development aid: per-phase SM cycle counters of the solver kernels, summed over CTAs.
 * enable=1 allocates/zeroes them, 0 frees; out (may be NULL) receives 26 values: the 14 dual-form phases below,
 * the 10 condensed-kernel phases {structure, block inverses, assembly of K, LU, solve: right-hand
 * side, solve: substitution, solve: back-substitution of the multipliers, residuals, step rules, gradients}
 * (the banded kernel's in the same slots), then two counts summed over every forward kernel that ran: the KKT
 * factorisations and the KKT solves (one forward + one backward substitution each) it executed. The dual-form
 * phases:
 * {prefactor, load T, LU, KKT solves, residuals, step rules,
 *  LU: diagonal blocks (look-ahead warp), LU: panel solves, LU: trailing updates,
 *  LU: diagonal-block inverses, number of diagonal blocks with row interchanges, number of
 *  diagonal blocks, LU: look-ahead warp's panel pieces + block update, LU: other warps waiting
 *  for the look-ahead warp}. */
int lcpb200_profile(lcpb200_handle_t h, int enable, long long* out);

/* LCPFunction.forward. Outputs: zhat[B,n], nu[B,e] (NULL if e==0), lam[B,m],
 * slack[B,m], status[B] int32, iters[B] int32 (PDIPM iterations executed),
 * resid[B] (best residual, same dtype; may be NULL), Rsave[B,m,m] (may be NULL):
 * the Schur matrix R = G Q^-1 G^T + F - ... of every scene (the `self.R` the
 * reference keeps for backward, lcp.py:28); pass it to lcpb200_backward to skip
 * the re-factorisation of Q and the Schur GEMM there. */
int lcpb200_forward(lcpb200_handle_t h, int B,
                    const void* Q, const void* p, const void* G, const void* hvec,
                    const void* A, const void* b, const void* F,
                    double eps, int not_improved_lim, int max_iter,
                    void* zhat, void* nu, void* lam, void* slack,
                    int32_t* status, int32_t* iters, void* resid, void* Rsave,
                    void* stream);

/* LCPFunction.backward. Inputs: the forward inputs it needs (Q,G,A,F), the
 * saved forward results (zhat, nu, lam, slack) and dl_dzhat[B,n].
 * Outputs (any may be NULL = skip): dQ[B,n,n] dp[B,n] dG[B,m,n] dh[B,m]
 * dA[B,e,n] db[B,e] dF[B,m,m]. */
int lcpb200_backward(lcpb200_handle_t h, int B,
                     const void* Q, const void* G, const void* A, const void* F,
                     const void* zhat, const void* nu, const void* lam, const void* slack,
                     const void* dl_dzhat,
                     void* dQ, void* dp, void* dG, void* dh, void* dA, void* db, void* dF,
                     const void* Rsave /* from lcpb200_forward, or NULL = recompute */,
                     unsigned flags, void* stream);

/* lcpb200_backward_batched: R >= 1 cotangents of the same saved solves in one call -- the rows of a
 * vector-Jacobian product (R = n one-hot cotangents per scene: the whole Jacobian of zhat). Same inputs as
 * lcpb200_backward, but dl_dzhat is [R,B,n] and every output is [R,B,...] or NULL (dQ[R,B,n,n], dp[R,B,n], ...):
 * slot r holds exactly what lcpb200_backward returns for dl_dzhat[r]. Each scene's KKT matrix is factored once
 * per chunk of cotangents, not once per cotangent; a scene's cotangents are split into chunks only to fill the GPU
 * when B is small, and the results do not depend on that split. Flags, Rsave and LCPB200_BWD_REUSE_STRUCTURE as
 * for lcpb200_backward, and the same kernel family serves each scene (fp32: condensed, the dual form for
 * unstructured scenes; fp64: the dual form, the condensed kernel for scenes whose dual LU broke down;
 * LCPB200_DUAL_BACKWARD=1: the dual form first for fp32 too). lcpb200_backward is this call with R = 1. */
int lcpb200_backward_batched(lcpb200_handle_t h, int R, int B,
                             const void* Q, const void* G, const void* A, const void* F,
                             const void* zhat, const void* nu, const void* lam, const void* slack,
                             const void* dl_dzhat,
                             void* dQ, void* dp, void* dG, void* dh, void* dA, void* db, void* dF,
                             const void* Rsave, unsigned flags, void* stream);

/* lcpb200_jvp_batched: R >= 1 Jacobian-vector products of the same saved solves in one call -- the forward-mode
 * derivative of zhat along R directions of (Q, p, G, h, A, b, F) (R = 1: one torch.func.jvp; R = k: the k columns
 * of a jacfwd). Same inputs and saved solve as lcpb200_backward_batched; every tangent is [R,B,...] with the shape
 * of its input (tQ[R,B,n,n], tp[R,B,n], tG[R,B,m,n], th[R,B,m], tA[R,B,e,n], tb[R,B,e], tF[R,B,m,m]) or NULL,
 * which means zero and is not read. dz[R,B,n] receives the tangents of zhat. Each scene's KKT matrix K (not
 * transposed) is factored once per chunk of tangents at the saved iterate, with each kernel family's d (the
 * condensed kernel clamps d = lam / slack to [1e-10, 1e10] in fp64, the dual form does not), so the result is the
 * transpose of the LCPB200_BWD_EXACT_ADJOINT backward: the true derivative of the solve. tQ enters as tQ zhat, as
 * given: the backward returns the symmetrised dQ, so the two agree along symmetric tQ. Scenes are routed as in
 * lcpb200_backward_batched. flags: 0 or LCPB200_BWD_REUSE_STRUCTURE. */
int lcpb200_jvp_batched(lcpb200_handle_t h, int R, int B,
                        const void* Q, const void* G, const void* A, const void* F,
                        const void* zhat, const void* nu, const void* lam, const void* slack,
                        const void* tQ, const void* tp, const void* tG, const void* th,
                        const void* tA, const void* tb, const void* tF,
                        void* dz, const void* Rsave, unsigned flags, void* stream);

/* Same two calls with HOST buffers: copies in, solves, copies out. The timed
 * "e2e" path of bench.py. Synchronous on return. forward_host leaves its inputs,
 * results and R on the device; backward_host with Q == NULL (then G, A, F, zhat,
 * nu, lam, slack are ignored) reuses them instead of uploading them again -- the
 * save_for_backward of lcp.py:34. Any other call on the handle drops that state. */
int lcpb200_forward_host(lcpb200_handle_t h, int B,
                         const void* Q, const void* p, const void* G, const void* hvec,
                         const void* A, const void* b, const void* F,
                         double eps, int not_improved_lim, int max_iter,
                         void* zhat, void* nu, void* lam, void* slack,
                         int32_t* status, int32_t* iters, void* resid);
int lcpb200_backward_host(lcpb200_handle_t h, int B,
                          const void* Q, const void* G, const void* A, const void* F,
                          const void* zhat, const void* nu, const void* lam, const void* slack,
                          const void* dl_dzhat,
                          void* dQ, void* dp, void* dG, void* dh, void* dA, void* db, void* dF,
                          unsigned flags);

/* Contact detection for B scenes of nb circles, np DYNAMIC convex polygons (the reference's Rect / Hull bodies) and no
 * static convex polygon obstacles (walls, floors, ramps: no degrees of freedom), replacing the pair loop of
 * World.find_contacts (physics/world.py:139-142), and, in the same call, the geometry and material of the selected
 * pairs for callers that do not differentiate through the contact generation. The pairs (i, j), i < j, of the body
 * list [circles 0..nb-1, polygons nb..nb+np-1, obstacles nb+np..nb+np+no-1] (obstacles never pair with each other) are
 * visited in lexicographic order, the contact order of a reference World built from [Circle..., Rect / Hull...,
 * pinned Rect / Hull...]. A pair gives 0, 1 or 2 contacts, stored in that order:
 *   circle-circle                 the circle-circle test of physics/contacts.py:68-80: a pair is a contact iff
 *                                 rad_i + rad_j - |pos_i - pos_j| >= -eps; geometry (contacts.py:69-77):
 *                                 normal = (pos1 - pos2) / dist, penetration = r1 + r2 - dist,
 *                                 p1 = -normal (r1 - pen / 2), p2 = normal (r2 - pen / 2);
 *   circle-polygon / -obstacle    the circle-hull rule of physics/contacts.py:84-144 with the exact closest point:
 *                                 centre outside, contact iff |c - q| - r <= eps (q the closest point of the polygon),
 *                                 normal = (c - q) / |c - q|, p1 = q - c, p2 = q - oref, penetration = r - |c - q|;
 *                                 centre inside, the edge of largest separation sep (outward unit normal n):
 *                                 normal = n, p1 = -n sep, p2 = c + p1 - oref, penetration = r - sep; oref is a
 *                                 dynamic polygon's centroid (a two-body contact) or an obstacle's reference point (a
 *                                 one-body contact);
 *   polygon-polygon / -obstacle   the hull-hull rule of physics/contacts.py:145-292: SAT both ways (edge normal
 *                                 left_orthogonal(e) / |e|, support with >=, the last maximal vertex wins; separated iff
 *                                 the largest edge separation is > eps; body2 holds the reference face iff its
 *                                 separation is strictly larger), the incident edge at the support vertex whose
 *                                 normal has the smallest dot product with the reference normal, and clipping of the
 *                                 incident edge to the planes +-|e_ref| / 2 about the REFERENCE BODY's CENTROID (not
 *                                 the edge's midpoint), twice, a point kept iff n . (v - v_ref) <= eps -- 0 to 2
 *                                 contacts, in the order of the clipped points. SAT scans start at edge 0 (the reference
 *                                 starts at the edge that won last time): the results differ only on an exact tie
 *                                 between two edge separations.
 * Zero-length edges (a vertex repeated to pad a polygon to nv) are skipped everywhere. mu / restitution of a contact
 * are the mean of the two bodies' (world.py:144-151, :213-224).
 * Device pointers (NULL allowed for an empty group):
 *   pos[B,nb,2] rad[B,nb] fric[B,nb] rest[B,nb]       circles (fric / rest: only for the geometry)
 *   pverts[B,np,nv,2] pcen[B,np,2] pfric[B,np] prest[B,np]
 *                                                     polygons: world-frame vertices (positive shoelace area),
 *                                                     centroids, friction and restitution
 *   overts[B,no,nv,2] oref[B,no,2] ofric[B,no] orest[B,no]
 *                                                     obstacles: world-frame vertices (convex, either orientation),
 *                                                     reference points (p2 is relative to it), friction and
 *                                                     restitution (ofric / orest: only for the geometry)
 *   body1[B,cap] body2[B,cap] int32                   OUT: the contacts' pairs in the order above (the order the
 *                                                     reference appends contacts in), padded with the pair (0, 1)
 *                                                     ((0, 0) when nb + np + no == 1);
 *                                                     body2 >= nb + np names obstacle body2 - nb - np, the one-body
 *                                                     contacts of lcpb200_engine_forward
 *   counts[B] int32                                   OUT: number of contacts (may exceed cap: then the lists hold the
 *                                                     first cap contacts and the caller must grow cap)
 *   feat[B,cap] int32                                 OUT: per hull-hull contact its discrete features (bits 0-1 the
 *                                                     point: incident endpoint 0 / 1, cut by the first / second clip
 *                                                     plane; bits 2-3 the first clip's outcome; bit 4 body2 holds the
 *                                                     reference face; bits 5-12 reference edge; bits 13-20 incident
 *                                                     edge), from which the geometry is rebuilt; -1 for other
 *                                                     contacts and unused slots (0 in unused slots when nb == 0:
 *                                                     a hull-hull padding pair). Required when np > 0 or
 *                                                     no_contact != NULL, NULL
 *                                                     allowed otherwise
 *   normal[B,cap,2] p1 p2[B,cap,2] penetration mu restitution_c[B,cap]
 *                                                     OUT, all NULL (detection only) or all non-NULL: geometry and
 *                                                     material of the selected pairs (penetration -1e30 in unused
 *                                                     slots)
 *   no_contact                                        NULL, or const uint32_t[ceil(nt * nt / 32)], shared by the batch:
 *                                                     bit i * nt + j (bit k is bit k % 32 of word k / 32), i < j,
 *                                                     nt = nb + np + no, set iff the pair (i, j) of the body list
 *                                                     never makes contact (the reference's Body.add_no_contact:
 *                                                     contacts.py:60 returns before any rule when
 *                                                     `geom1 in geom2.no_contact`). Only bits with i < j are read; a
 *                                                     pair of two obstacles is never visited anyway. An excluded pair
 *                                                     gives no contact and no rule is evaluated for it.
 * 3 <= nv <= 256 when np + no > 0; oref is required when no > 0. The walk follows the arguments: with no_contact, the
 * polygon walk reading the mask; else with feat, the polygon walk; else (np == 0) the circle walk, at most one contact
 * per pair. With np == 0 the pairs, their order and the geometry do not depend on which walk runs. */
int lcpb200_contacts(int dtype, int B, int nb, int np, int no, int nv, int cap, double eps, const void* pos,
                     const void* rad, const void* fric, const void* rest, const void* pverts, const void* pcen,
                     const void* pfric, const void* prest, const void* overts, const void* oref, const void* ofric,
                     const void* orest, int32_t* body1, int32_t* body2, int32_t* counts, int32_t* feat, void* normal,
                     void* p1, void* p2, void* penetration, void* mu, void* restitution_c,
                     const uint32_t* no_contact, void* stream);

/* lcpb200_contacts for a batch whose scenes hold different bodies: scene s takes part with the bodies whose bit is set
 * in active[s] and walks the pairs of those bodies only, so its contact list is that of the world holding just its
 * active bodies (same rules, same lexicographic order, body indices of the full list) and its walk costs its own
 * pairs. The arguments are those of lcpb200_contacts, plus:
 *   no_contact                                        NULL, or per-scene pair masks in the layout of lcpb200_contacts:
 *                                                     scene s reads the mask at no_contact + s * no_contact_stride
 *                                                     (in uint32 words; stride 0: one mask shared by the batch), with
 *                                                     the bit of the pair's body indices
 *   active[B, ceil(nt / 32)] uint32                   NULL (every body active), or bit k % 32 of word k / 32 of row s
 *                                                     set iff body k of [circles, polygons, obstacles] is active in
 *                                                     scene s; bits at k >= nt are ignored
 * feat is required; nt = nb + np + no <= 8192 (the active list of a scene is kept in shared memory), else an error.
 * Padding pairs and feat of unused slots are those of lcpb200_contacts. With every body active and a shared mask the
 * outputs equal lcpb200_contacts'. */
int lcpb200_contacts_active(int dtype, int B, int nb, int np, int no, int nv, int cap, double eps, const void* pos,
                            const void* rad, const void* fric, const void* rest, const void* pverts, const void* pcen,
                            const void* pfric, const void* prest, const void* overts, const void* oref,
                            const void* ofric, const void* orest, int32_t* body1, int32_t* body2, int32_t* counts,
                            int32_t* feat, void* normal, void* p1, void* p2, void* penetration, void* mu,
                            void* restitution_c, const uint32_t* no_contact, long long no_contact_stride,
                            const uint32_t* active, void* stream);

/* Ray casts against the bodies of B scenes (the body groups of lcpb200_contacts): R rays per scene, each an origin and a
 * UNIT direction (not normalised here), cast against the body list [circles 0..nb-1, polygons nb..nb+np-1, obstacles
 * nb+np..nb+np+no-1] at their current pose. A ray hits a body only where it ENTERS it at some 0 <= t <= max_dist:
 *   circle (c, r)                 w = o - c, b = u . w, k = |w|^2 - r^2: a miss if k < 0 (the origin is inside),
 *                                 b >= 0 or disc = b^2 - k < 0, else t = k / (-b + sqrt(disc)); feat -1, normal
 *                                 (o + t u - c) / r
 *   polygon / obstacle            convex, either orientation; Cyrus-Beck clipping against every edge of non-zero length
 *                                 (outward unit normal n_e, start vertex v_e, num = n_e . (v_e - o), den = n_e . u):
 *                                 den == 0 a miss if num < 0, else the edge is ignored; den < 0 an entering edge at
 *                                 t = num / den, the largest wins (the first edge on a tie); den > 0 a leaving edge,
 *                                 the smallest t kept. A hit iff an entering edge exists and 0 <= t_enter <= t_leave,
 *                                 t_enter <= max_dist; feat = the entering edge, normal = its n_e. An origin inside the
 *                                 polygon gives t_enter < 0: no hit.
 * The nearest hit wins; an exact tie goes to the lower body index. A ray that hits nothing gets body -1, feat -1,
 * t = max_dist and a zero normal; so does a direction of zero length or with a non-finite component, or a non-finite
 * origin. Deterministic (no atomics); results do not depend on how the rays are split into CTAs.
 * Device pointers:
 *   pos[B,nb,2] rad[B,nb]                             circles (NULL when nb == 0)
 *   pverts[B,np,nv,2] overts[B,no,nv,2]               polygons and obstacles: world-frame vertices (NULL when the
 *                                                     group is empty); a vertex repeated to pad to nv is skipped
 *   origin[B,R,2] dir[B,R,2]                          the rays; dir of unit length
 *   active_words[B, ceil(nt / 32)] int32              NULL (every body visible), or the layout of lcpb200_contacts_active:
 *                                                     bit k % 32 of word k / 32 of row s set iff body k is active in
 *                                                     scene s; inactive bodies are invisible (nt <= 8192)
 *   t[B,R] body[B,R] feat[B,R] int32                  OUT: distance, body index (-1: no hit), entering edge (-1: a
 *                                                     circle or no hit)
 *   normal[B,R,2]                                     OUT or NULL: the surface normal at the hit
 * Returns non-zero without launching on B <= 0, R <= 0, nb + np + no == 0, nv > 256 (or nv < 3 with polygons),
 * max_dist < 0 or non-finite (in the dtype), a NULL required pointer, active_words with nt > 8192, or B * R > 2^31 - 1. */
int lcpb200_raycast(int dtype, int B, int nb, int np, int no, int nv, int R, double max_dist, const void* pos,
                    const void* rad, const void* pverts, const void* overts, const void* origin, const void* dir,
                    const int32_t* active_words, void* t, int32_t* body, int32_t* feat, void* normal, void* stream);

/* Signed distances from query points to the bodies of B scenes (the body groups of lcpb200_contacts): Q points per
 * scene (or Q points shared by every scene), each tested against the body list [circles 0..nb-1, polygons
 * nb..nb+np-1, obstacles nb+np..nb+np+no-1] at their current pose; inactive bodies are skipped.
 *   circle (c, r)                 sdf = |x - c| - r, feat -1, normal (x - c) / |x - c|; (0, 0) when x == c
 *   polygon / obstacle            convex, either orientation; every edge of non-zero length e (start vertex v_e, end
 *                                 vertex v_f, E = v_f - v_e, outward unit normal n_e) gives s_e = n_e . (x - v_e).
 *                                 Inside (every s_e <= 0): sdf = max_e s_e, feat = 256 + e of the largest (the first
 *                                 edge on a tie), normal n_e. Outside: t = clamp((x - v_e) . E / |E|^2, 0, 1), closest
 *                                 point q_e = v_e if t <= 0, v_f (the vertex itself, not v_e + E) if t >= 1, else
 *                                 v_e + t E; sdf = min_e |x - q_e| (the first edge on a tie: the two edges meeting at a
 *                                 vertex tie exactly in its region), feat = e, normal (x - q) / |x - q|.
 * The smallest sdf wins; an exact tie goes to the lower body index (from best = max_dist, body -1, a body replaces the
 * best iff body < 0 ? sdf <= best : sdf < best). A point with no body at sdf <= max_dist, or a non-finite point, gets
 * body -1, feat -1, sdf = max_dist and a zero normal. This is the exact Euclidean signed distance of one circle or
 * convex polygon; for overlapping bodies it is the min of theirs, exact outside every body and a bound inside.
 * Deterministic (no atomics); results do not depend on how the points are split into CTAs.
 * Device pointers:
 *   pos[B,nb,2] rad[B,nb]                             circles (NULL when nb == 0)
 *   pverts[B,np,nv,2] overts[B,no,nv,2]               polygons and obstacles: world-frame vertices (NULL when the
 *                                                     group is empty); a vertex repeated to pad to nv is skipped
 *   points[B,Q,2], or [Q,2] with shared_points = 1    the query points; shared_points = 1: every scene reads the same Q
 *   active_words[B, ceil(nt / 32)] int32              NULL (every body present), or the layout of
 *                                                     lcpb200_contacts_active (nt <= 8192); inactive bodies are skipped
 *   sdf[B,Q] body[B,Q] feat[B,Q] int32                OUT: signed distance, body index (-1: none within max_dist),
 *                                                     feature (-1: a circle or none; e: outside, nearest edge e;
 *                                                     256 + e: inside, nearest face e)
 *   normal[B,Q,2]                                     OUT or NULL: the unit direction of increasing distance
 * Returns non-zero without launching on B <= 0, Q <= 0, nb + np + no == 0, nv > 256 (or nv < 3 with polygons),
 * max_dist < 0 or non-finite (in the dtype), a NULL required pointer, active_words with nt > 8192, or B * Q > 2^31 - 1. */
int lcpb200_signed_distance(int dtype, int B, int nb, int np, int no, int nv, int Q, double max_dist, const void* pos,
                            const void* rad, const void* pverts, const void* overts, const void* points,
                            int shared_points, const int32_t* active_words, void* sdf, int32_t* body, int32_t* feat,
                            void* normal, void* stream);

/* Distances between bodies of B scenes (the body groups of lcpb200_contacts), K queries per scene (or K queries shared
 * by every scene). Every pair (A, B) reduces to the signed distance of one feature point of one body (the source: a
 * circle's centre, radius r, or a polygon's vertex, r = 0) to the other body (the target), minus r. Target distances
 * and choices are those of lcpb200_signed_distance (feat -1 circle, e outside / nearest edge e, 256 + e face e):
 *   circle i - circle j         source the centre of i: d = |c_i - c_j| - r_j - r_i
 *   circle - polygon            source the circle's centre (either order): d = sdf(centre, polygon) - r
 *   polygon - polygon           S = max over the faces e of both polygons of min over the other's vertices v of
 *                               n_e . (v - v_e) (A's faces win a tie; either orientation, zero-length padding edges
 *                               skipped). S > 0 (separated): d is the exact Euclidean distance, min over A's vertices
 *                               of their outside distance to B and over B's vertices of theirs to A (the first vertex
 *                               wins a tie, A's before B's), target feat e. S <= 0 (overlapping or touching): d = S,
 *                               the minimum translation distance; source the support vertex of the SAT face (the last
 *                               maximal vertex), target feat 256 + e.
 * normal is the unit normal n from A towards B (moving B along n increases d): minus the target's sdf normal at the
 * source when A is the source, that normal when B is; zero where the source is the target's closest point. point_a is
 * the witness on A; point_b = point_a + d n is the witness on B. When separated both lie on the boundaries and
 * |point_b - point_a| = d; when overlapping one is the support vertex and the other its projection onto the SAT face's
 * supporting line, which need not lie on the face segment.
 * Pair mode (body_b != NULL): query k reads the pair (body_a[k], body_b[k]) and body[k] = body_b[k] on a hit. Nearest
 * mode (body_b == NULL): query k reads body_a[k] and finds the nearest other active body of its scene, obstacles
 * included, skipping the pairs of no_contact; candidates in index order, from best = max_dist, body -1, a body
 * replaces the best iff body < 0 ? d <= best : d < best. A hit iff d <= max_dist. A query whose body is inactive or out
 * of range, that names one body twice, or with nothing within max_dist reads dist = max_dist, body -1, feat -1 and
 * zero normal and point_a. Deterministic (no atomics); results do not depend on how the queries are split into CTAs.
 * Device pointers:
 *   pos[B,nb,2] rad[B,nb] pverts[B,np,nv,2] overts[B,no,nv,2]   the bodies, as in lcpb200_signed_distance
 *   body_a[B,K] int32, or [K] with shared_queries = 1  the first body of each pair, or the query body (nearest mode)
 *   body_b[B,K] int32, or [K] with shared_queries = 1  the second body of each pair; NULL: nearest mode
 *   active_words[B, ceil(nt / 32)] int32              NULL, or the layout of lcpb200_contacts_active (nt <= 8192)
 *   no_contact, nc_stride                             NULL, or the pair masks of lcpb200_contacts_active (bit
 *                                                     i * nt + j for i < j; scene s at no_contact + s * nc_stride,
 *                                                     nc_stride 0: one mask shared by the batch); nearest mode only
 *   dist[B,K] body[B,K] feat[B,K] int32               OUT: distance, the other body (-1: a miss), and the choices:
 *                                                     bits 0-8 the target's sdf feat (e or 256 + e; 0 for a circle
 *                                                     target), bits 9-16 the source vertex (0 for a circle), bit 17
 *                                                     set iff B is the source; -1 on a miss
 *   normal[B,K,2] point_a[B,K,2]                      OUT: n and the witness on A
 * Returns non-zero without launching on B <= 0, K <= 0, nb + np + no == 0, nv > 256 (or nv < 3 with polygons),
 * max_dist < 0 or non-finite (in the dtype), a NULL required pointer (body_a, the bodies, every output),
 * nc_stride < 0, active_words with nt > 8192, or B * K > 2^31 - 1. */
int lcpb200_body_distance(int dtype, int B, int nb, int np, int no, int nv, int K, double max_dist, const void* pos,
                          const void* rad, const void* pverts, const void* overts, const int32_t* body_a,
                          const int32_t* body_b, int shared_queries, const int32_t* active_words,
                          const int32_t* no_contact, long long nc_stride, void* dist, int32_t* body, int32_t* feat,
                          void* normal, void* point_a, void* stream);

/* Shape casts and translational sweeps against the bodies of B scenes (the body groups of lcpb200_contacts), K queries
 * per scene. Every case reduces to one cast primitive: a ray from a point x along a unit direction s u (s = +-1)
 * against a target feature inflated by a radius rho >= 0, hitting at the first entry into the Minkowski sum of the
 * target and a disk of radius rho (the minimum t >= 0 over the target's features):
 *   circle (c, R)                 the ray against the circle (c, R + rho), lcpb200_raycast's rule: w = x - c,
 *                                 b = s u . w, k = |w|^2 - (R + rho)^2, a hit iff k >= 0, b < 0 and b^2 - k >= 0, at
 *                                 t = k / (-b + sqrt(b^2 - k)); normal m = (w + t s u) / (R + rho); feat 0
 *   polygon face e                every edge of non-zero length (outward unit normal n_e, start vertex v_e, E the
 *                                 edge): the offset line n_e . (y - v_e) = rho, a hit iff den = n_e . s u < 0,
 *                                 t = (n_e . (v_e - x) + rho) / den >= 0 and the hit point projects onto the edge
 *                                 within [0, 1] (inclusive); m = n_e; feat e
 *   polygon vertex v (rho > 0)    the circle (v, rho) with the circle rule; m = (x + t s u - v) / rho; feat 256 + v
 * Within a polygon the faces come first, then the vertices, each in index order, and only a strictly nearer hit
 * replaces the best. A target the swept shape overlaps at t = 0 is skipped; one it only touches gives t = 0 when the
 * motion heads into it and no hit otherwise.
 * Disk mode (body_q == NULL): query k sweeps a disk of radius radius[k] from origin[k] along dir[k] against every
 * active body: x = origin, s = +1, rho = radius; a polygon is skipped when its signed distance at the origin (the rule
 * of lcpb200_signed_distance) is < radius. A hit iff t <= max_dist. no_contact and limit are not read.
 * Body mode (body_q != NULL): query k translates body q = body_q[k] along dir[k] by at most limit[k] against every other
 * active body of its scene not excluded by no_contact, held still (no rotation):
 *   circle q, circle j            x = c_q, s = +1, the circle j with rho = R_q
 *   circle q, polygon j           x = c_q, s = +1, polygon j with rho = R_q (skipped when sdf(c_q, j) < R_q)
 *   polygon q, circle j           x = c_j, s = -1, polygon q at its current pose with rho = R_j (skipped when
 *                                 sdf(c_j, q) < R_j): the mover is the target
 *   polygon q, polygon j          every vertex of q with s = +1 against j, then every vertex of j with s = -1 against
 *                                 q, rho = 0 (q's vertices first, the first strictly nearest wins); skipped when the
 *                                 separating-axis value of both polygons, taken both ways, is < 0
 * Candidates in index order, from best = the limit (max_dist in disk mode), body -1: a body replaces the best iff
 * body < 0 ? t <= best : t < best. A miss -- nothing hit, a zero or non-finite direction, a non-finite origin or limit,
 * a negative or non-finite radius, an inactive or out-of-range mover -- reads dist = the limit, body -1, feat -1 and
 * zero normal and point. Deterministic (no atomics); results do not depend on how the queries are split into CTAs.
 * Device pointers:
 *   pos[B,nb,2] rad[B,nb] pverts[B,np,nv,2] overts[B,no,nv,2]   the bodies, as in lcpb200_signed_distance
 *   origin[B,K,2] radius[B,K]                         disk mode: the disks (NULL in body mode)
 *   body_q[B,K] int32                                 body mode: the movers; NULL: disk mode
 *   dir[B,K,2]                                        the unit directions (not normalised here)
 *   limit[B,K]                                        body mode: the length of each translation (NULL in disk mode)
 *   active_words[B, ceil(nt / 32)] int32              NULL, or the layout of lcpb200_contacts_active (nt <= 8192)
 *   no_contact, nc_stride                             NULL, or the pair masks of lcpb200_body_distance; body mode only
 *   dist[B,K] body[B,K] feat[B,K] int32               OUT: t, the hit body (-1: a miss), and the choices: bits 0-8 the
 *                                                     target feature, bits 9-16 the source vertex (0 for a circle
 *                                                     source), bit 17 set iff the source is the hit body (the mover
 *                                                     is the target); -1 on a miss
 *   normal[B,K,2]                                     OUT: disk mode, the hit body's outward normal m at the contact;
 *                                                     body mode, the unit normal from the mover towards the hit body
 *                                                     (-m, or m when the mover is the target)
 *   point[B,K,2]                                      OUT: the contact point at the time of impact, x + s t u - R_src m
 *                                                     plus t u when the mover is the target (R_src: the source
 *                                                     circle's radius, 0 for a polygon vertex)
 * The radius is not read on the host: a negative or non-finite one reads a miss. Returns non-zero without launching on
 * B <= 0, K <= 0, nb + np + no == 0, nv > 256 (or nv < 3 with polygons), max_dist < 0 or non-finite (in the dtype), a
 * NULL pointer the mode reads (dir, origin and radius or limit, the bodies, every output), nc_stride < 0, active_words
 * with nt > 8192, or B * K > 2^31 - 1. */
int lcpb200_shapecast(int dtype, int B, int nb, int np, int no, int nv, int K, double max_dist, const void* pos,
                      const void* rad, const void* pverts, const void* overts, const void* origin, const void* radius,
                      const int32_t* body_q, const void* dir, const void* limit, const int32_t* active_words,
                      const int32_t* no_contact, long long nc_stride, void* dist, int32_t* body, int32_t* feat,
                      void* normal, void* point, void* stream);

/* Times of impact between bodies that translate and rotate over a step, in B scenes (the body groups of
 * lcpb200_contacts), K queries per scene. Over tau in [0, 1] dynamic body k moves as p_k + tau motion_k, motion =
 * (dth, dx, dy) in the layout of p: a circle's centre moves (its rotation is irrelevant), a polygon's vertices are
 * c + tau dc + R(tau dth)(v - c) (v its vertices, c its centre at tau = 0), obstacles stay. d(tau) is the body distance
 * of lcpb200_body_distance between the two bodies at their poses at tau.
 * Conservative advancement from tau = 0: at each iterate, with d = d(tau), its unit normal n (from A towards B) and
 *   mu = -n . (dc_B - dc_A) + |dth_A| R_A + |dth_B| R_B      (R: the largest |v - c| of a polygon, 0 otherwise)
 * a hit at tau iff d - gap <= tol; no hit iff mu <= 0 or tau + (d - gap) / mu > 1; else tau += (d - gap) / mu. mu bounds
 * how fast d can fall, so the reported tau is never later than the first time d reaches gap. At most 64 evaluations:
 * a pair that reaches the cap reports the tau it reached as a hit (dist then shows d - gap > tol). A pair with
 * d(0) < skip is not seen, one with d(0) == skip only when mu > 0; nor is a pair whose bodies do not move or one with a
 * non-finite motion row.
 * Pair mode (body_b != NULL): query k is the pair (body_a[k], body_b[k]); a pair naming one body twice or an inactive
 * body misses. First mode (body_b == NULL): query k is body_a[k] against every other active body of its scene not
 * excluded by no_contact (the candidates of lcpb200_body_distance's nearest mode), in index order, from best = 1, body
 * -1: a body replaces the best iff body < 0 ? tau <= best : tau < best. Deterministic (no atomics); results do not
 * depend on how the queries are split into CTAs.
 * Device pointers:
 *   pos[B,nb,2] rad[B,nb] pverts[B,np,nv,2] overts[B,no,nv,2]   the bodies at tau = 0, as in lcpb200_signed_distance
 *   pcen[B,np,2]                                      the polygons' centres c (NULL when np == 0)
 *   motion[B,nb+np,3]                                 (dth, dx, dy) per dynamic body (NULL when nb + np == 0)
 *   body_a[B,K] / body_b[B,K] int32                   as in lcpb200_body_distance ([K] when shared_queries != 0)
 *   active_words, no_contact, nc_stride               as in lcpb200_body_distance; no_contact is read in first mode
 *   frac[B,K] body[B,K] feat[B,K] int32               OUT: tau (1 on a miss), the hit body (-1: a miss) and the pair's
 *                                                     dist_feat at tau (lcpb200_body_distance's packing; -1 on a miss)
 *   dist[B,K]                                         OUT: d at tau (0 on a miss)
 *   normal[B,K,2] point_a[B,K,2]                      OUT: n and the witness on A at tau, world coordinates (zero on a
 *                                                     miss); the witness on B is point_a + dist normal
 * gap >= 0 is the distance that counts as contact, skip >= 0 the overlap threshold above, tol >= 0 the tolerance of
 * the stop. Returns non-zero without launching on B <= 0, K <= 0, nb + np + no == 0, nv > 256 (or nv < 3 with
 * polygons), gap, skip or tol negative or non-finite (in the dtype), a NULL required pointer (body_a, the bodies,
 * pcen, motion, every output), nc_stride < 0, active_words with nt > 8192, or B * K > 2^31 - 1. */
int lcpb200_time_of_impact(int dtype, int B, int nb, int np, int no, int nv, int K, double gap, const void* pos,
                           const void* rad, const void* pverts, const void* overts, const void* pcen,
                           const void* motion, const int32_t* body_a, const int32_t* body_b, int shared_queries,
                           double skip, double tol, const int32_t* active_words, const int32_t* no_contact,
                           long long nc_stride, void* frac, int32_t* body, int32_t* feat, void* dist, void* normal,
                           void* point_a, void* stream);

/* Contact-list -> dense LCP assembly for B scenes of nb bodies (3 dofs each,
 * n = 3 nb), nc contacts, fd = 2 friction directions (world.py:191-192),
 * m = nc (2 + fd). Structure-of-arrays inputs:
 *   mass[B,nb] inertia[B,nb] v[B,n] fext[B,n]           bodies
 *   normal[B,nc,2] p1[B,nc,2] p2[B,nc,2]                contact geometry
 *   body1[nc] body2[nc] int32 (shared by the batch)     contact topology
 *   mu[B,nc] restitution[B,nc]                          contact material
 * Outputs: Q[B,n,n] p[B,n] G[B,m,n] h[B,m] F[B,m,m]  with
 *   p = M v + dt fext,  h = [(Jc v) restitution, 0, 0]  (engines.py:32,53,74). */
int lcpb200_assemble(int dtype, int B, int nb, int nc, double dt,
                     const void* mass, const void* inertia, const void* v, const void* fext,
                     const void* normal, const void* p1, const void* p2,
                     const int32_t* body1, const int32_t* body2,
                     const void* mu, const void* restitution,
                     void* Q, void* p, void* G, void* hvec, void* F, void* stream);

/* Adjoint of lcpb200_assemble: given dQ dp dG dh dF, accumulate gradients
 * w.r.t. mass, inertia, v, fext, normal, p1, p2, mu, restitution (any NULL = skip). */
int lcpb200_assemble_backward(int dtype, int B, int nb, int nc, double dt,
                              const void* mass, const void* inertia, const void* v,
                              const void* normal, const void* p1, const void* p2,
                              const int32_t* body1, const int32_t* body2,
                              const void* mu, const void* restitution,
                              const void* dQ, const void* dp, const void* dG,
                              const void* dh, const void* dF,
                              void* dmass, void* dinertia, void* dv, void* dfext,
                              void* dnormal, void* dp1, void* dp2,
                              void* dmu, void* drestitution, void* stream);

/* Fused engine entry points (SURVEY.md 8(b): lcpb200_assemble_solve). They replace, in ONE kernel per pass,
 *   mode 0: PdipmEngine.solve_dynamics' LCP (physics/engines.py:50-76) incl. the assembly of
 *           world.py:144-234:  zhat = LCP(M, M v + dt f, [Jc; Jf; 0], [(Jc v) rest, 0, 0], A, b, F(E, mu));
 *           the engine returns -zhat (engines.py:76);
 *   mode 1: PdipmEngine.post_stabilization's LCP (physics/engines.py:80-116):
 *           zhat = LCP(M, 0, Jc, (Jc v)(1 - rest), A, b, 0).
 * Inputs are the contact structure-of-arrays of lcpb200_assemble (+ optional equality rows A[B,e,n], b[B,e],
 * e.g. World.Je()); nothing dense is written to or read from HBM. The handle must have been created with
 * n = 3 nb, m = 4 nc (mode 0) or nc (mode 1). n + e <= 128: the condensed-KKT kernels (fp32 / fp64); larger
 * scenes (fp64 only, e.g. BASELINE config 4: 512 bodies): the banded large-scene kernels (lcp_banded.cuh), which
 * order the bodies so that the condensed matrix is an arrow matrix (<= 16 border rows: pinned bodies, bodies with
 * > 12 two-body contacts, equality rows) whose half bandwidth bw, rounded up to a multiple of 8, is at most the
 * plan's limit. That limit comes from shared memory: on an H100 it is 128 rows up to 773 bodies, 120 up to 1492,
 * 112 up to 2173 and 104 beyond (a half bandwidth of 42, 39, 36, 34 bodies). A scene whose contact topology the kernel
 * cannot take (a contact of a body with itself, > 16 contacts on one body for the condensed kernels, a band or
 * border beyond the limits above) gets status -100 and no result: assemble it with lcpb200_assemble and call
 * lcpb200_forward.
 * Static obstacles: body2[c] >= nb names a body without degrees of freedom (a wall, floor or ramp: the static
 * obstacles of lcpb200_contacts). Contact c is then a ONE-BODY contact: its rows of G touch body1's three
 * columns only, exactly the reference's formulation with the obstacle pinned by a TotalConstraint, reduced by the
 * pinned dofs. p2 is not used by such a contact and its dp2 gradient is zero. body1 must be < nb; body1 == body2, a
 * negative index or a body1 >= nb gets status -100.
 * contact_count == NULL: every scene has the nc contacts body1[nc], body2[nc] (one topology for the batch).
 * contact_count[B] != NULL (batched worlds): scene s uses its first contact_count[s] <= nc contacts, body1 /
 * body2 are [B,nc] and all per-contact arrays are strided by nc; a scene with 0 contacts gets the
 * equality-constrained solve of engines.py:35-49; lam / slack rows of scene s are laid out for ITS count
 * (normal rows [0,c), friction [c,3c), gamma [3c,4c)), the arrays keep the stride m.
 * lcpb200_engine_backward: the chain rule through the assembly applied to the factored gradients of
 * lcp.py:52-63 (dG = dlam (x) zhat + lam (x) dx, ...): gradients w.r.t. the contact list, any may be NULL.
 * flags: LCPB200_BWD_BUG_COMPATIBLE (the reference's gradients) or LCPB200_BWD_EXACT_ADJOINT (the true
 * adjoint: the transposed KKT system), on both the condensed and the large-scene kernels. */
int lcpb200_engine_forward(lcpb200_handle_t h, int B, int nb, int nc, int mode, double dt,
                           const void* mass, const void* inertia, const void* v, const void* fext,
                           const void* normal, const void* p1, const void* p2,
                           const int32_t* body1, const int32_t* body2, const int32_t* contact_count,
                           const void* mu, const void* restitution, const void* A, const void* b,
                           double eps, int not_improved_lim, int max_iter,
                           void* zhat, void* nu, void* lam, void* slack,
                           int32_t* status, int32_t* iters, void* resid, void* stream);
int lcpb200_engine_backward(lcpb200_handle_t h, int B, int nb, int nc, int mode, double dt,
                            const void* mass, const void* inertia, const void* v, const void* fext,
                            const void* normal, const void* p1, const void* p2,
                            const int32_t* body1, const int32_t* body2, const int32_t* contact_count,
                            const void* mu, const void* restitution, const void* A,
                            const void* zhat, const void* nu, const void* lam, const void* slack,
                            const void* dl_dzhat,
                            void* dmass, void* dinertia, void* dv, void* dfext,
                            void* dnormal, void* dp1, void* dp2, void* dmu, void* drestitution,
                            void* dA, void* db, unsigned flags, void* stream);
/* lcpb200_engine_backward_batched: R >= 1 cotangents of the same saved solves in one call -- the rows of a
 * vector-Jacobian product, e.g. R = n one-hot cotangents for the whole Jacobian of zhat. Same inputs as
 * lcpb200_engine_backward (one set for the batch: mass[B,nb], ..., zhat[B,n], lam / slack[B,m], nu[B,e]), but
 * dl_dzhat is [R,B,n] and every output is [R,B,...] (dmass[R,B,nb], dv[R,B,n], dnormal[R,B,nc,2], dA[R,B,e,n],
 * ...): slot r holds exactly what lcpb200_engine_backward returns for the cotangent dl_dzhat[r]. Each scene's
 * KKT matrix is factored once per chunk of cotangents, not once per cotangent; the cotangents of a scene are split
 * into chunks only to fill the GPU when B is small, and the results do not depend on that split. The same NULL
 * rules and flags as lcpb200_engine_backward; a scene with status -100 gets zero gradients in every slot.
 * lcpb200_engine_backward is this call with R = 1. */
/* lcpb200_engine_jvp_batched: R >= 1 Jacobian-vector products of the same saved solves in one call -- the
 * forward-mode derivative of zhat along R directions of the inputs (R = 1: one torch.func.jvp; R = k: the k columns
 * of a jacfwd). Same primal inputs and saved solve as lcpb200_engine_backward_batched; every tangent is [R,B,...]
 * with the shape of its input (t_mass[R,B,nb], t_v[R,B,n], t_normal[R,B,nc,2], t_A[R,B,e,n], t_b[R,B,e], ...) or
 * NULL, which means zero and is not read. dz[R,B,n] receives the tangents of zhat. Each scene's KKT matrix K (not
 * transposed) is factored once per chunk of tangents at the backward's d clamp, so the result is the transpose of
 * the LCPB200_BWD_EXACT_ADJOINT backward: the true derivative of the solve. A scene with status -100 gets zero
 * rows. Same kernel selection as the backward (the large-scene kernel when the condensed one cannot take the
 * sizes, or LCPB200_FORCE_BANDED=1 for fp64). */
int lcpb200_engine_jvp_batched(lcpb200_handle_t h, int R, int B, int nb, int nc, int mode, double dt,
                               const void* mass, const void* inertia, const void* v, const void* fext,
                               const void* normal, const void* p1, const void* p2,
                               const int32_t* body1, const int32_t* body2, const int32_t* contact_count,
                               const void* mu, const void* restitution, const void* A,
                               const void* zhat, const void* nu, const void* lam, const void* slack,
                               const void* t_mass, const void* t_inertia, const void* t_v, const void* t_fext,
                               const void* t_normal, const void* t_p1, const void* t_p2, const void* t_mu,
                               const void* t_restitution, const void* t_A, const void* t_b,
                               void* dz, void* stream);
int lcpb200_engine_backward_batched(lcpb200_handle_t h, int R, int B, int nb, int nc, int mode, double dt,
                                    const void* mass, const void* inertia, const void* v, const void* fext,
                                    const void* normal, const void* p1, const void* p2,
                                    const int32_t* body1, const int32_t* body2, const int32_t* contact_count,
                                    const void* mu, const void* restitution, const void* A,
                                    const void* zhat, const void* nu, const void* lam, const void* slack,
                                    const void* dl_dzhat,
                                    void* dmass, void* dinertia, void* dv, void* dfext,
                                    void* dnormal, void* dp1, void* dp2, void* dmu, void* drestitution,
                                    void* dA, void* db, unsigned flags, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* LCPB200_H */
