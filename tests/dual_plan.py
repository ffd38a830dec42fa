"""Host restatement of the dual-form kernels' plan (csrc/lcpb200.cu `make_plan`) and of the branches their kernels
take per scene (csrc/lcp_solver.cuh), no GPU.

* `make_plan` restates `make_plan` (lcpb200.cu:96-160) with `pad_ld` (:87-94) and `Vecs::carve`
  (lcp_solver.cuh:55-72): the padded row count mp, the threads per CTA, where T lives (mode 0: shared memory,
  1: split with U12 in L2, 2: L2), m1 / ldT / ldL, the staging leading dimension of G, where G and Q^-1 live, the
  dynamic shared memory and the per-CTA workspace regions, for a given opt-in shared-memory limit.
  `describe` is the dual-form part of `lcpb200_describe` (:309-314) without the grid.
* `verdict` restates the per-scene branches: qdiag and singular Q (`prefactor`, lcp_solver.cuh:409-429), the
  R-forming branch (:431-465: staged Gram, unstaged Gram, general GEMM), the ELL copy of F (`build_f_ell`, 4 per
  row), the ELL copies of G (`build_g_ell`: only for G in L2, 8 per row and 32 per column), the prefetch of R
  (`prefetch_T`, :489-511: not in mode 2, m % VC == 0, R 16-byte aligned) and the first diagonal block factored
  beside the residuals (:862: the prefetch, not mode 2, mp == m).
* Scene builders (plain float64 torch): the engine's contact scenes (tests/cond_plan.py's `assemble`), dense
  random scenes, a non-diagonal SPD Q, a chosen number of non-zeros in one F row, one G row or one G column,
  a singular Q, and a scene with a non-finite right-hand side.
"""
import functools

import torch

from tests import cond_plan as cp

H100_SMEM_OPTIN = 232448          # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100
F_ELL, G_ELL_ROW, G_ELL_COL = 4, 8, 32
MODES = ("smem", "smem-split(U12 in L2)", "L2")


def blk(ts):
    """LU block size NB (Blk<T>)."""
    return 32 if ts == 4 else 16


def vc(ts):
    """Elements per 16-byte vector (VecOf<T>::VC)."""
    return 16 // ts


def al4(x):
    return (x + 3) & ~3


def pad_ld(cols, ts):
    """Leading dimension >= cols: a multiple of the 16-byte vector and == 4 (mod 32) in 32-bit words."""
    wpe = ts // 4
    ld = cols
    while (ld * wpe) % 32 != 4 or (ld * ts) % 16 != 0:
        ld += 1
    return ld


def vec_elems(n, mp, e, nt, nb):
    """Vecs::carve: elements of the shared-memory vectors."""
    sizes = [n, mp, mp, e, mp,                 # x s z y d
             n, mp, e,                         # rx rz ry
             mp, e, e,                         # hz hy te
             n, n,                             # tn tn2
             n, mp, mp, e,                     # dxa dsa dza dya
             n, mp, mp, e,                     # dxc dsc dzc dyc
             mp, n, nb * (nb + 4) + nb,        # rs2 qinv lt
             max(4 * nt, mp), 128, mp,         # scratch red perm
             2 * (nb + 4), 4, mp, 4]           # stage bcast rdiag iflag
    return sum(al4(s) for s in sizes)


@functools.lru_cache(maxsize=None)
def make_plan(ts, n, m, e, optin=H100_SMEM_OPTIN):
    """The plan of a handle for sizeof(T) = ts, or None when the shared-memory vectors alone exceed the limit
    (lcpb200_create then fails, or serves the engine entry points only)."""
    NB, VC = blk(ts), vc(ts)
    mp = -(-m // NB) * NB
    nt = 512 if (mp >= 96 or n >= 96) else (256 if mp >= 64 else 128)
    vec = vec_elems(n, mp, e, nt, NB)
    budget = optin - 1024 - vec * ts
    if budget < 0:
        return None
    off = 0
    ldfull = pad_ld(mp, ts)
    n2 = tiles = 0
    if mp * ldfull * ts <= budget:
        mode, m1, ldT, ldL = 0, mp, ldfull, 0
        off += al4(mp * ldfull)
    else:
        m1 = -(-(mp // 2) // NB) * NB
        n2 = mp - m1
        ldl = pad_ld(m1, ts)
        tiles = -(-n2 // 16) * -(-n2 // (16 * VC))
        need = (m1 * ldfull + n2 * ldl) * ts
        if 0 < n2 <= m1 and need <= budget and tiles <= nt // 32:
            mode, ldT, ldL = 1, ldfull, ldl
            off += al4(m1 * ldfull) + al4(n2 * ldl)
        else:
            mode, m1, ldT, ldL, n2, tiles = 2, mp, -(-mp // VC) * VC, 0, 0, 0
    stage_ld = 0
    if mode != 2:
        lds = pad_ld(n, ts)
        if m * lds <= m1 * ldT:
            stage_ld = lds
    budget -= off * ts
    ldQi = -(-n // VC) * VC
    Gb, Qb = al4(m * n), al4(n * ldQi)
    G_smem = Qi_smem = False
    if Gb * ts <= budget:
        G_smem = True
        off += Gb
        budget -= Gb * ts
    if Qb * ts <= budget:
        Qi_smem = True
        off += Qb
        budget -= Qb * ts
    ws = []                                        # per-CTA L2 workspace regions (name, elements), in order
    ws.append(("Qi", Qb))
    ws.append(("R", al4(m * m)))
    ws.append(("T", al4(mp * ldT) if mode == 2 else 0))
    ws.append(("U12", al4(m1 * (mp - m1)) if mode == 1 else 0))
    ws.append(("X", al4(n * m)))
    ws.append(("XA", al4(n * e)))
    ws.append(("S11", al4(e * e)))
    ws.append(("V", al4(m * e)))
    ws.append(("W", al4(e * m)))
    ws.append(("Fell", al4(m * 8)))
    ws.append(("Gell", al4(16 * m + 64 * n)))
    regions, o = {}, 0
    for name, size in ws:
        regions[name] = (o, size)
        o += size
    return dict(ts=ts, n=n, m=m, e=e, mp=mp, nt=nt, mode=mode, m1=m1, n2=mp - m1, ldT=ldT, ldL=ldL, tiles=tiles,
                stage_ld=stage_ld, G_smem=G_smem, Qi_smem=Qi_smem, smem_bytes=(off + vec) * ts, ws_per_cta=o,
                regions=regions, vec_elems=vec)


def describe(plan):
    """The dual-form part of Handle.describe() (up to the grid, which depends on the GPU's SM count)."""
    return "dual: threads=%d smem=%dB T:%s m1=%d ldT=%d ldL=%d G:%s Qinv:%s" % (
        plan["nt"], plan["smem_bytes"], MODES[plan["mode"]], plan["m1"], plan["ldT"], plan["ldL"],
        "smem" if plan["G_smem"] else "L2", "smem" if plan["Qi_smem"] else "L2")


def tier(plan):
    """(nt, mode, G residency, Q^-1 residency, staged) -- the tier a shape falls in."""
    return (plan["nt"], plan["mode"], "smem" if plan["G_smem"] else "L2", "smem" if plan["Qi_smem"] else "L2",
            plan["stage_ld"] > 0)


# ------------------------------------------------------------------------------------------ per-scene branches
def _nnz_rows(M):
    return int((M != 0).sum(-1).max()) if M.numel() else 0


def verdict(Q, G, F, plan, r_aligned=True, transF=False):
    """The branches the dual-form kernels take for one scene (Q [n,n], G [m,n], F [m,m]) under `plan`.
    r_aligned: R's address is 16-byte aligned (always on the device path; the host pipeline's saved R of scene k
    sits at k m^2 elements). Returns dict(qdiag, singular, rform, f_ell, g_ell, prefetch, overlap)."""
    Q, G, F = (torch.as_tensor(t, dtype=torch.float64) for t in (Q, G, F))
    ts, n, m = plan["ts"], plan["n"], plan["m"]
    qd = torch.diagonal(Q)
    qdiag = not bool((Q - torch.diag(qd)).ne(0).any())
    singular = qdiag and not bool(((qd != 0) & torch.isfinite(qd)).all())
    if not qdiag or n % vc(ts) != 0:
        rform = "gemm"
    elif plan["mode"] != 2 and plan["stage_ld"] > 0:
        rform = "staged"
    else:
        rform = "unstaged"
    if plan["G_smem"]:
        g_ell = "n/a"                       # G is copied into shared memory: the dense GEMVs read it there
    else:
        g_ell = _nnz_rows(G) <= G_ELL_ROW and _nnz_rows(G.t()) <= G_ELL_COL
    prefetch = plan["mode"] != 2 and m % vc(ts) == 0 and r_aligned
    return dict(qdiag=qdiag, singular=singular, rform=rform, f_ell=_nnz_rows(F.t() if transF else F) <= F_ELL,
                g_ell=g_ell, prefetch=prefetch, overlap=prefetch and plan["mp"] == m)


def verdicts(inp, plan, **kw):
    Q, p, G, h, A, b, F = inp
    return [verdict(Q[s], G[s], F[s], plan, **kw) for s in range(Q.shape[0])]


# ------------------------------------------------------------------------------------------ scenes
def sizes(inp):
    Q, p, G, h, A, b, F = inp
    return Q.shape[1], G.shape[1], (A.shape[1] if A.dim() > 1 else 0)


def engine_scenes(B, nb, nc, fd=2, e=0, seed=0):
    """The engine's contact scenes (n = 3 nb, m = nc (2 + fd)) on scenes.pile_layout's pile."""
    return cp.contact_scenes(B, nb, nc, fd, e=e, seed=seed)


def dense_scenes(B, n, m, e=0, seed=0):
    """Fully dense SPD Q, G and F (scenes.make_dense_random)."""
    from lcp_physics_b200.scenes import make_dense_random
    return make_dense_random(B, n, m, e=e, dtype=torch.float64, seed=seed)


def nondiag_q(inp, scale=0.05):
    """Q with symmetric couplings between neighbouring dofs (still SPD: the engine's masses are >= 0.2, so Q stays
    diagonally dominant): the kernels invert Q densely and form R by the general GEMMs."""
    Q, p, G, h, A, b, F = [t.clone() for t in inp]
    n = Q.shape[1]
    i = torch.arange(n - 1)
    Q[:, i, i + 1] += scale
    Q[:, i + 1, i] += scale
    return Q, p, G, h, A, b, F


def singular_q(inp, scenes):
    """A zero mass in Q of the given scenes: status -1, NaN results."""
    Q, p, G, h, A, b, F = [t.clone() for t in inp]
    for s in scenes:
        Q[s, 1, 1] = 0
    return Q, p, G, h, A, b, F


def nonfinite_h(inp, scenes):
    """A NaN in h of the given scenes: every iterate of that scene is NaN (status 1 after not_improved_lim + 1
    iterations), including whatever the triangular solves write into the padded tails of the vectors."""
    Q, p, G, h, A, b, F = [t.clone() for t in inp]
    for s in scenes:
        h[s, 0] = float("nan")
    return Q, p, G, h, A, b, F


def _fill(M, idx, scale):
    """Set M[..., i] = scale (1 + 0.1 i) for every i in idx where M is zero (every scene)."""
    for i in idx:
        M[..., i] = torch.where(M[..., i] == 0, torch.full_like(M[..., i], scale * (1 + 0.1 * (i % 7))), M[..., i])


def f_row_nnz(inp, row, k, scale=0.02):
    """F with exactly k non-zeros in `row` in every scene (small entries added in the first zero columns)."""
    Q, p, G, h, A, b, F = [t.clone() for t in inp]
    have = (F[0, row] != 0).nonzero().flatten().tolist()
    assert all(bool((F[s, row] != 0).sum() == len(have)) for s in range(F.shape[0])) and len(have) <= k
    free = [j for j in range(F.shape[1]) if j not in have][:k - len(have)]
    row_v = F[:, row]
    _fill(row_v, free, scale)
    F[:, row] = row_v
    return Q, p, G, h, A, b, F


def g_row_nnz(inp, row, k, scale=0.02):
    """G with exactly k non-zeros in `row` in every scene."""
    Q, p, G, h, A, b, F = [t.clone() for t in inp]
    have = (G[0, row] != 0).nonzero().flatten().tolist()
    assert all(bool((G[s, row] != 0).sum() == len(have)) for s in range(G.shape[0])) and len(have) <= k
    free = [j for j in range(G.shape[2]) if j not in have][:k - len(have)]
    row_v = G[:, row]
    _fill(row_v, free, scale)
    G[:, row] = row_v
    return Q, p, G, h, A, b, F


def g_col_nnz(inp, col, k, scale=0.02):
    """G with exactly k non-zeros in column `col` in every scene: entries added in zero rows, last rows first (the
    engine's gamma rows, which are zero in G), so that no row passes G_ELL_ROW."""
    Q, p, G, h, A, b, F = [t.clone() for t in inp]
    have = (G[0, :, col] != 0).nonzero().flatten().tolist()
    assert all(bool((G[s, :, col] != 0).sum() == len(have)) for s in range(G.shape[0])) and len(have) <= k
    zero_rows = [r for r in range(G.shape[1] - 1, -1, -1) if not bool((G[:, r] != 0).any())]
    free = zero_rows[:k - len(have)]
    assert len(free) == k - len(have), "not enough zero rows"
    col_v = G[:, :, col]
    _fill(col_v, free, scale)
    G[:, :, col] = col_v
    return Q, p, G, h, A, b, F


def cat(*inps):
    """Scenes of several batches (same sizes) in one batch."""
    out = []
    for parts in zip(*inps):
        out.append(torch.cat(parts, 0) if parts[0].dim() > 1 else parts[0])
    return tuple(out)
