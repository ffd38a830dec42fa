"""Host restatement of the condensed-KKT kernels' plan and admission rules (csrc/lcp_condensed.cuh), no GPU.

* `make_plan` restates `make_cplan` + `carve_plan` (lcpb200.cu / lcp_condensed.cuh): the block count NS, the
  capacities pcap and wcap, the shared-memory layout (the K region's floors: K itself, the structure scratch, the
  LU broadcast buffers and the SolveLayout) and the CTAs per SM, for a given opt-in shared-memory limit.
* `verdict_dense` restates `build_structure` (dense Q, G, F) and `verdict_soa` `build_structure_soa` (the engine's
  contact list): accepted, with the `Struct` (ncomp, cs, sh) and `mark_band_lu`'s choice, or rejected, with the
  rule that rejects it.
* `apply_grid_ok` is the invariant `comp_apply` needs: its U positions per thread cover the grid t < cs << sh
  (U = 4 before it was sized per cs, `old=True`).
* Scene builders (plain float64 torch): contact scenes with fd friction directions (cs = 2 + fd), cs = 2 and
  cs = 1 components, mixed sizes, one-body rows, and scenes just inside and just outside every limit.
"""
import functools
import math

import numpy as np
import torch

from tests import band_plan as bp

NT, UC, CSMAX, KS, LMAX, LU_BW = 256, 8, 6, 8, 16, 2
H100_SMEM_OPTIN = 232448          # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100
SM_SMEM = 228 * 1024              # shared memory per SM
NS_SIZES = (2, 3, 4, 6, 8)


def al16(x):
    return (x + 15) & ~15


def ceil_log2(x):
    sh = 0
    while (1 << sh) < x:
        sh += 1
    return sh


def apply_span(cs, old=False):
    """Positions per thread of comp_apply<CS> (ApplySpan<CS>::U)."""
    if old:
        return 4
    return -(-(cs << ceil_log2(4 * NT // cs)) // NT)


def scratch_bytes(n, m, ts):
    return (al16(2 * KS * m * 2) + al16(2 * KS * m * ts) + al16(5 * m * 4) + al16(CSMAX * m * 2) + al16(8 * m * 4)
            + al16(LMAX * n * 2) + al16(n * 4) + 64)


def carve(n, m, e, NS, pcap, wcap, ts):
    """carve_plan: total dynamic shared memory of the layout."""
    NP = 16 * NS
    qn = (NP + 31) // 32
    kb = max(NP * NP * 8, scratch_bytes(n, m, ts), 8 * NP * 8, (NP // qn) * qn * qn * 32 * 8)
    sizes = [kb, wcap * 8, pcap * 8, NP * 8, NP * 8, wcap * ts, UC * pcap * ts, e * n * ts]
    sizes += [n * ts] * 4 + [e * ts] * 3 + [m * ts] * 7 + [192 * ts]
    sizes += [pcap * 2, m * 2, LMAX * n * 2, UC * pcap, pcap, n, 16 * 4]
    return sum(al16(s) for s in sizes)


@functools.lru_cache(maxsize=None)
def make_plan(ts, n, m, e, optin=H100_SMEM_OPTIN):
    """make_cplan for sizeof(T) = ts: dict(NS, NP, pcap, wcap, smem_bytes, ctas_per_sm), or None (no condensed
    plan: the dense API takes the dual form for every scene, the engine path the banded kernel / an error)."""
    N = n + e
    if N > 128 or n > 255 or m > 4 * NT:
        return None
    NS = min(s for s in NS_SIZES if 16 * s >= N)
    pcap = (m + 7) & ~7
    dyn_max = optin - 1024
    target = 2 if NS <= 6 else 1
    for want in range(target, 0, -1):
        lim = min(dyn_max, SM_SMEM // want - 1024 - 64)
        for mult in range(CSMAX, 0, -1):
            wcap = mult * pcap
            smem = carve(n, m, e, NS, pcap, wcap, ts)
            if smem <= lim:
                return dict(n=n, m=m, e=e, NS=NS, NP=16 * NS, pcap=pcap, wcap=wcap, mult=mult, smem_bytes=smem,
                            ctas_per_sm=want)
            if mult <= 4:
                break
    return None


def tsize(dtype):
    return 4 if dtype == torch.float32 else 8


def apply_grid_ok(st, old=False):
    return (st["cs"] << st["sh"]) <= apply_span(st["cs"], old) * NT


# ------------------------------------------------------------------------------------------ verdicts
def _components(Fpat):
    """Connected components of F's sparsity graph (both directions), rows in increasing order."""
    m = Fpat.shape[0]
    label = list(range(m))

    def find(i):
        while label[i] != i:
            label[i] = label[label[i]]
            i = label[i]
        return i
    for i, j in zip(*np.nonzero(Fpat)):
        a, b = find(int(i)), find(int(j))
        if a != b:
            label[max(a, b)] = min(a, b)
    comps = {}
    for i in range(m):
        comps.setdefault(find(i), []).append(i)
    return list(comps.values())


def _struct(ncomp, cs, cols, e):
    wide = e > 0 or any(c and (c[-1] >> 4) - (c[0] >> 4) > LU_BW for c in cols)
    return dict(ok=True, rule=None, ncomp=ncomp, cs=cs, sh=ceil_log2(ncomp), band_lu=not wide)


def verdict_dense(Q, G, F, e, plan):
    """build_structure for one scene (Q [n,n], G [m,n], F [m,m]) under `plan` (make_plan's dict, or None).
    Returns dict(ok, rule, ncomp, cs, sh, band_lu); rule names the failed check: 'plan', 'singular' (status -1),
    'Q', 'KS', 'm', 'CSMAX', 'pcap', 'wcap', 'UC', 'LMAX'."""
    Q, G, F = (np.asarray(t, dtype=np.float64) for t in (Q, G, F))
    if plan is None:
        return dict(ok=False, rule="plan")
    qd = np.diag(Q)
    if not np.all((qd != 0) & np.isfinite(qd)):
        return dict(ok=False, rule="singular")
    if np.count_nonzero(Q - np.diag(qd)):
        return dict(ok=False, rule="Q")
    if (F != 0).sum(1).max(initial=0) > KS or (G != 0).sum(1).max(initial=0) > KS:
        return dict(ok=False, rule="KS")
    m = G.shape[0]
    if m > 4 * NT:
        return dict(ok=False, rule="m")
    comps = _components(F != 0)
    ncomp, cs = len(comps), max(len(c) for c in comps)
    for rule, bad in (("CSMAX", cs > CSMAX), ("pcap", ncomp * cs > plan["pcap"]), ("wcap", ncomp * cs * cs > plan["wcap"])):
        if bad:
            return dict(ok=False, rule=rule, ncomp=ncomp, cs=cs)
    cols = [sorted(set(np.nonzero(G[c].any(0))[0].tolist())) for c in comps]
    if max(len(c) for c in cols) > UC:
        return dict(ok=False, rule="UC", ncomp=ncomp, cs=cs)
    per_col = np.zeros(G.shape[1], dtype=int)
    for c in cols:
        per_col[c] += 1
    if per_col.max(initial=0) > LMAX:
        return dict(ok=False, rule="LMAX", ncomp=ncomp, cs=cs)
    return _struct(ncomp, cs, cols, e)


def verdict_soa(nb, body1, body2, nc_stride, mode, e, plan, count=None):
    """build_structure_soa for one scene: body1 / body2 [nc_stride] ints, count = this scene's contacts (default all).
    Masses are assumed non-zero. Rules: 'plan', 'count', 'pcap', 'wcap', 'topology', 'LMAX'."""
    if plan is None:
        return dict(ok=False, rule="plan")
    cs = 4 if mode == 0 else 1
    nc = nc_stride if count is None else int(count)
    if nc < 0 or nc > nc_stride or cs * nc > plan["m"]:
        return dict(ok=False, rule="count")
    if nc * cs > plan["pcap"]:
        return dict(ok=False, rule="pcap")
    if nc * cs * cs > plan["wcap"]:
        return dict(ok=False, rule="wcap")
    per_col = np.zeros(3 * nb, dtype=int)
    cols = []
    for c in range(nc):
        b1, b2 = int(body1[c]), int(body2[c])
        if b1 == b2 or b1 < 0 or b2 < 0 or b1 >= nb:
            return dict(ok=False, rule="topology")
        bodies = sorted((b1, b2)) if b2 < nb else [b1]
        cc = [3 * b + q for b in bodies for q in range(3)]
        per_col[cc] += 1
        cols.append(cc)
    if per_col.max(initial=0) > LMAX:
        return dict(ok=False, rule="LMAX")
    return _struct(nc, cs, cols, e)


# ------------------------------------------------------------------------------------------ scenes
def _dirs(normal, fd, gen):
    """Friction directions of assemble_dense: +-left_orthogonal(n), then independent random directions."""
    d1 = torch.stack([normal[..., 1], -normal[..., 0]], -1)
    dirs = [d1, -d1][:fd]
    for _ in range(fd - len(dirs)):
        a = torch.rand(normal.shape[:-1], generator=gen, dtype=torch.float64) * (2 * math.pi)
        dirs.append(torch.stack([torch.cos(a), torch.sin(a)], -1))
    return dirs


def assemble(soa, fd=2, e=0, dt=1.0 / 30, gravity=10.0, seed=0):
    """(Q, p, G, h, A, b, F) of scenes.assemble_dense for any fd >= 0 (cs = 2 + fd rows per contact), with one-body
    contacts (body2 >= nb: rows touch body1's columns only). fd = 0: a normal row and a gamma row per contact."""
    mass, inertia = soa["mass"], soa["inertia"]
    B, nb = mass.shape
    f64 = torch.float64
    normal, p1, p2 = soa["normal"], soa["p1"], soa["p2"]
    nc = normal.shape[1]
    i1, i2 = soa["body1"].long(), soa["body2"].long()
    two = i2 < nb
    i2c = torch.where(two, i2, torch.zeros_like(i2))
    n, m = 3 * nb, nc * (2 + fd)
    Md = torch.stack([inertia, mass, mass], -1).reshape(B, n)
    Q = torch.diag_embed(Md)
    cross = lambda a, b: a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]
    ar = torch.arange(nc)

    def rows(d):
        J = torch.zeros(B, nc, n, dtype=f64)
        J[:, ar, 3 * i1] += cross(p1, d)
        J[:, ar, 3 * i1 + 1] += d[..., 0]
        J[:, ar, 3 * i1 + 2] += d[..., 1]
        w = two.to(f64)
        J[:, ar, 3 * i2c] -= w * cross(p2, d)
        J[:, ar, 3 * i2c + 1] -= w * d[..., 0]
        J[:, ar, 3 * i2c + 2] -= w * d[..., 1]
        return J

    Jc = rows(normal)
    gen = torch.Generator().manual_seed(seed + 7919)
    dirs = _dirs(normal, fd, gen)
    Jf = torch.stack([rows(d) for d in dirs], 2).reshape(B, nc * fd, n) if fd else torch.zeros(B, 0, n, dtype=f64)
    G = torch.cat([Jc, Jf, torch.zeros(B, nc, n, dtype=f64)], 1)
    E = torch.zeros(nc * fd, nc, dtype=f64)
    for k in range(fd):
        E[torch.arange(nc) * fd + k, torch.arange(nc)] = 1
    F = torch.zeros(B, m, m, dtype=f64)
    F[:, nc:nc + nc * fd, nc + nc * fd:] = E
    F[:, nc + nc * fd:, :nc] = torch.diag_embed(soa["mu"])
    F[:, nc + nc * fd:, nc:nc + nc * fd] = -E.t()
    fvec = torch.zeros(B, n, dtype=f64)
    fvec[:, 2::3] = gravity * mass
    p = Md * soa["v"] + dt * fvec
    h = torch.cat([torch.bmm(Jc, soa["v"].unsqueeze(2)).squeeze(2) * soa["restitution"],
                   torch.zeros(B, nc * fd + nc, dtype=f64)], 1)
    if e > 0:
        A = torch.zeros(B, e, n, dtype=f64)
        A[:, torch.arange(e), torch.arange(e)] = 1
        b = torch.zeros(B, e, dtype=f64)
    else:
        A = b = torch.tensor([], dtype=f64)
    return Q, p, G, h, A, b, F


def pile(B, nb, nc, seed=0):
    """scenes.make_contact_soa: a jittered grid pile (its contact list is shared by the batch)."""
    from lcp_physics_b200.scenes import make_contact_soa
    return make_contact_soa(B, nb, nc, seed=seed)


def contact_scenes(B, nb, nc, fd, e=0, seed=0):
    """Contact scenes with fd friction directions on scenes.pile_layout's pile: components of cs = 2 + fd rows."""
    return assemble(pile(B, nb, nc, seed), fd=fd, e=e, seed=seed)


def graph_soa(sc, B, seed=0):
    """Engine inputs (band_plan.to_soa) for B copies of a contact graph built by band_plan."""
    return bp.to_soa(sc, B=B, seed=seed)


def circulant(nb, nc, ks=(1, 2, 3, 4, 5, 6, 7, 8), radius=10.0):
    """nb bodies on a circle, contact c joins body i and i + k (mod nb) for k in ks, i fastest, first nc pairs:
    every body has degree <= 2 len(ks)."""
    pos = np.stack([radius * np.cos(2 * np.pi * np.arange(nb) / nb), radius * np.sin(2 * np.pi * np.arange(nb) / nb)], 1)
    pairs = [(i, (i + k) % nb) for k in ks for i in range(nb)][:nc]
    assert len(pairs) == nc
    return bp.contacts_from_positions(pos, pairs)


def cs2_scenes(B, nb, nc, seed=0):
    """cs = 2 components: a normal row coupled to one friction row through a monotone 2 x 2 block
    F_c = [[a, -b], [b, a]] (a > 0: positive definite symmetric part)."""
    soa = pile(B, nb, nc, seed)
    Q, p, G, h, A, b, F = assemble(soa, fd=1, seed=seed)          # rows [normal; friction; gamma]
    g = torch.Generator().manual_seed(seed + 1)
    a = torch.rand(B, nc, generator=g, dtype=torch.float64) * 0.5 + 0.5
    s = torch.rand(B, nc, generator=g, dtype=torch.float64) * 0.5
    ar = torch.arange(nc)
    F = torch.zeros(B, 2 * nc, 2 * nc, dtype=torch.float64)
    F[:, ar, ar] = a
    F[:, nc + ar, nc + ar] = a
    F[:, ar, nc + ar] = -s
    F[:, nc + ar, ar] = s
    return Q, p, G[:, :2 * nc].contiguous(), h[:, :2 * nc].contiguous(), A, b, F


def mixed_scenes(B, nb, nc, extra=1, seed=0):
    """Components of mixed sizes in one scene: the fd = 2 contact scene (cs = 4 components) with `extra` more rows,
    each a 1-row component (a copy of contact k's normal row, F_kk = 0.5), whose slots 1-3 are padding. The padded
    positions count against pcap (m rounded up to 8): with nc even, one extra row fits and three do not."""
    Q, p, G, h, A, b, F = contact_scenes(B, nb, nc, 2, seed=seed)
    m = 4 * nc
    G2 = torch.cat([G, G[:, :extra] * 0.9], 1)
    h2 = torch.cat([h, h[:, :extra]], 1)
    F2 = torch.zeros(B, m + extra, m + extra, dtype=torch.float64)
    F2[:, :m, :m] = F
    F2[:, m + torch.arange(extra), m + torch.arange(extra)] = 0.5
    return Q, p, G2.contiguous(), h2.contiguous(), A, b, F2


def floor_contacts(nb, nc):
    """nb bodies in a row, nc one-body contacts against a floor below them (body2 = nb), round robin over the
    bodies, each at its own point with a normal tilted by up to +-0.15 rad: no two rows are parallel."""
    pos = np.stack([np.arange(nb) * 3.0, np.zeros(nb)], 1)
    b1 = np.arange(nc) % nb
    per = -(-nc // nb)
    a = 0.3 * ((np.arange(nc) // nb) / max(per - 1, 1) - 0.5)
    nrm = np.stack([np.sin(a), -np.cos(a)], 1)
    off = 0.8 * ((np.arange(nc) // nb) / max(per - 1, 1) - 0.5)
    p1 = np.stack([off, np.ones(nc)], 1)
    return dict(nb=nb, pos=pos, body1=b1.astype(np.int32), body2=np.full(nc, nb, dtype=np.int32), normal=nrm, p1=p1,
                p2=np.zeros((nc, 2)))


def poststab_scenes(B, nb, nc, seed=0):
    """cs = 1: contact-normal rows only, F = 0 (the post-stabilisation LCP's structure)."""
    Q, p, G, h, A, b, F = contact_scenes(B, nb, nc, 2, seed=seed)
    return Q, p, G[:, :nc].contiguous(), h[:, :nc].contiguous(), A, b, torch.zeros(B, nc, nc, dtype=torch.float64)


def with_extra_g(inp, row, cols, scale=0.05):
    """A copy of the scenes with entries added to G[:, row, cols] (widens a row / its component's column set)."""
    Q, p, G, h, A, b, F = [t.clone() for t in inp]
    for c in cols:
        G[:, row, c] += scale * (1 + 0.1 * c)
    return Q, p, G, h, A, b, F


def one_body(nb, nc, n_obst):
    """Contact graph: scenes.pile_layout's pile of nb bodies with nc two-body contacts, plus n_obst one-body
    contacts against a floor (body2 = nb) on bodies 0, 1, ... in turn."""
    from lcp_physics_b200.scenes import pile_layout
    W, H, i1, i2 = pile_layout(nb, nc)
    k = np.arange(nb)
    pos = np.stack([(k % W) * 2.0 + 1e-3 * (k // W), (k // W) * 2.0], 1)
    obst = [(j % nb, 0.01) for j in range(n_obst)]
    return bp.contacts_from_positions(pos, list(zip(i1.tolist(), i2.tolist())), obst, floor_normal=(0.0, 1.0))


def dense_from_graph(sc, B, fd, e=0, seed=0):
    """Dense scenes (assemble) of B copies of a band_plan contact graph."""
    return assemble(graph_soa(sc, B, seed), fd=fd, e=e, seed=seed)


# ------------------------------------------------------------------------------------------ limits
def _widen(inp, rows_cols):
    """A copy of dense scenes with G[:, row, col] set for every (row, col) in rows_cols."""
    Q, p, G, h, A, b, F = [t.clone() for t in inp]
    for r, c in rows_cols:
        G[:, r, c] = 0.05 * (1 + 0.1 * c)
    return Q, p, G, h, A, b, F


def _base(seed):
    return contact_scenes(2, 16, 24, 2, seed=seed)       # contact 0 joins bodies 0 and 1 (columns 0-5)


# name -> (dtype, builder of the scene just inside, builder of the scene just outside), two scenes each (float64)
LIMIT_SCENES = {
    # a friction row of contact 0 with 8 / 9 entries (two / three columns of body 10 added)
    "KS_entries_per_row": (torch.float64, lambda: _widen(_base(81), [(24, 30), (24, 31)]),
                           lambda: _widen(_base(81), [(24, 30), (24, 31), (24, 32)])),
    # contact 0's component with 8 / 9 distinct columns, no row above 8 entries
    "UC_columns_per_component": (torch.float64, lambda: _widen(_base(82), [(24, 30), (25, 31)]),
                                 lambda: _widen(_base(82), [(24, 30), (24, 31), (25, 32)])),
    # components of 6 / 7 rows (4 / 5 friction directions)
    "CSMAX_rows_per_component": (torch.float64, lambda: contact_scenes(2, 16, 24, 4, seed=83),
                                 lambda: contact_scenes(2, 16, 24, 5, seed=83)),
    # a hub body in 16 / 17 contacts: 16 / 17 list entries in each of its columns
    "LMAX_entries_per_column": (torch.float64, lambda: dense_from_graph(bp.hubs(1, 16, ring=20), 2, 2, seed=84),
                                lambda: dense_from_graph(bp.hubs(1, 17, ring=20), 2, 2, seed=84)),
    # padded positions: one / three extra 1-row components next to 24 four-row ones (pcap = 104)
    "pcap_padded_positions": (torch.float64, lambda: mixed_scenes(2, 16, 24, extra=1, seed=85),
                              lambda: mixed_scenes(2, 16, 24, extra=3, seed=85)),
    # W and Fd entries: 146 / 147 five-row components on cfg 3's pile; make_cplan lowers wcap to 5 / 4 pcap
    "wcap_after_make_cplan": (torch.float32, lambda: contact_scenes(2, 32, 146, 3, seed=86),
                              lambda: contact_scenes(2, 32, 147, 3, seed=86)),
    # the shared memory: at n = 120 (NS = 8) fp64 plans reach 108 contacts (m = 432, wcap = 4 pcap), not 109
    "plan_shared_memory": (torch.float64, lambda: dense_from_graph(circulant(40, 108), 2, 2, seed=87),
                           lambda: dense_from_graph(circulant(40, 109), 2, 2, seed=87)),
}


def limit_scenes(name):
    dtype, inside, outside = LIMIT_SCENES[name]
    return dtype, inside(), outside()


def hub_world_record(sc, seed=0, fric=0.5, rest=0.3):
    """One world (helpers.ReplayWorld record) with the contact graph sc, uniform friction and restitution, and the
    dense LCP (assemble, fd = 2) the reference engine builds for it."""
    soa = graph_soa(sc, 1, seed)
    nc = len(sc["body1"])
    soa["mu"] = torch.full((1, nc), fric, dtype=torch.float64)
    soa["restitution"] = torch.full((1, nc), rest, dtype=torch.float64)
    Md = torch.stack([soa["inertia"], soa["mass"], soa["mass"]], -1).reshape(-1)
    rec = dict(t=0.0, M=torch.diag(Md).numpy(), Je=np.zeros((0, Md.numel())), v=soa["v"][0].numpy(),
               f=soa["fext"][0].numpy(), fric=np.full(sc["nb"], fric), rest=np.full(sc["nb"], rest),
               normal=sc["normal"], p1=sc["p1"], p2=sc["p2"], b1=sc["body1"], b2=sc["body2"])
    return rec, assemble(soa, fd=2)
