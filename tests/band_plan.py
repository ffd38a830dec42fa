"""Host restatement of the banded large-scene kernel's plan and ordering (csrc/lcp_banded.cuh), no GPU.

* `carve_plan` restates `carve_bplan`: the shared-memory layout, the widest supported active band `bwa_max` and
  the window size that is left over, for a given opt-in shared-memory limit.
* `order` restates `build_structure`: the border classification, the adjacency sorted by contact index, the
  warp-synchronous breadth-first sweeps, the coordinates integrated along the BFS tree, the x / y rank orderings
  and the choice of the narrowest of the three. It returns the sizes the kernel derives (nband, nbb, bwb,
  bw = 3 bwb + 2, bwa, Nbp).
* `admitted` is the kernel's admission rule: the border fits, bwa <= bwa_max, and the window fits the
  shared memory (`old=True`: the rule before bwa_max was enforced, window check only).
* Scene builders (contact lists with geometry): degree-capped random graphs, lattices, hexagonal piles and hubs.
  Every contact sits at the midpoint of its two bodies (p1 = -d/2 n, p2 = d/2 n, n = (x1 - x2) / d), so the
  coordinates the kernel integrates along its BFS tree are the bodies' positions.
"""
import math

import numpy as np
import torch

NT, BD, PV, DEGB = 256, 16, 8, 12
H100_SMEM_OPTIN = 232448          # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100
SUBR_ROWS = 4 * 32                # rows one substitution pass updates (SUBR = 4 rounds of 32 lanes)


def _r16(x):
    return (x + 15) & ~15


def dyn_limit(optin=H100_SMEM_OPTIN):
    """Dynamic shared memory the plan may use (lcpb200.cu: opt-in limit - 1024)."""
    return optin - 1024


def carve_plan(nb, ncap, cs, optin=H100_SMEM_OPTIN):
    """carve_bplan for n = 3 nb: dict(bwa_max, win_bytes, ldk, fbs, LP, g_FB_end, ...) or None (does not fit)."""
    limit = dyn_limit(optin)
    n = 3 * nb
    nbp = (n + 7) & ~7
    o = 0
    for size in (6 * 32 * 8, 64 * 4, nb * 4, BD * BD * 8, (nbp + BD) * 8):   # red, sv, rank, cf, sol
        o += _r16(size)
    fixed = o
    best = 0
    for bwa in range(8, 129, 8):
        ldw = bwa + PV + BD + 1
        need = fixed + 2 * (bwa + BD) * PV * 8 + 32 + ldw * ldw * 8
        if need > limit:
            break
        best = bwa
    if best == 0:
        return None
    o += 2 * _r16((best + BD) * PV * 8)                                     # lp, up
    win_bytes = (limit - o) & ~15
    if (3 * nb + 1 + 2 * ncap) * 4 + 8 + 28 * nb > win_bytes:
        return None
    return dict(nb=nb, n=n, nbp=nbp, fixed=fixed, bwa_max=best, win_bytes=win_bytes, win_doubles=win_bytes // 8,
                ldk=best + 1, LP=best + BD, fbs=72 + 2 * PV * (best + BD), smem_bytes=o + win_bytes)


def band_sizes(bwb):
    """Sizes build_structure derives from the ordered half bandwidth bwb (in bodies)."""
    bw = 3 * bwb + 2
    bwa = (bw + 7) & ~7
    Wc = bwa + PV
    return dict(bw=bw, bwa=bwa, Wc=Wc, LDW=Wc + BD + 1, LP=bwa + BD, fbs=72 + 2 * PV * (bwa + BD), ldk=bw + 1)


def admitted(plan, bwb, nbd=0, old=False):
    """build_structure's verdict (True = solved, False = status -100) for a scene ordered to bwb with a
    border of nbd = 3 nbb + e rows."""
    if nbd > BD:
        return False
    s = band_sizes(bwb)
    if not old and s["bwa"] > plan["bwa_max"]:
        return False
    return s["LDW"] * s["LDW"] <= plan["win_doubles"]


def fits_plan(plan, bwb):
    """Every per-pass array the plan sized holds the band: Kb / KbT rows, the two panels, the factor blocks
    and the substitution's rows."""
    s = band_sizes(bwb)
    return (s["ldk"] <= plan["ldk"] and s["LP"] <= plan["LP"] and s["fbs"] <= plan["fbs"]
            and s["bwa"] <= SUBR_ROWS)


# ------------------------------------------------------------------------------------------ ordering
def order(nb, b1, b2, p1, p2, A=None):
    """build_structure's ordering of one scene. b1, b2: [nc] ints (b2 >= nb: a static obstacle); p1, p2: [nc, 2]
    float64 contact points; A: optional [e, 3 nb] equality rows. Returns a dict with nband, nbb, nbd, bwb, bw,
    bwa, Nbp, the chosen candidate (0 = BFS, 1 = x, 2 = y), the per-candidate widths and rank[nb] (band
    position, or -1 - border index)."""
    b1 = [int(v) for v in b1]
    b2 = [int(v) for v in b2]
    nc = len(b1)
    p1 = np.asarray(p1, dtype=np.float64).reshape(nc, 2).tolist()
    p2 = np.asarray(p2, dtype=np.float64).reshape(nc, 2).tolist()
    e = 0 if A is None else int(A.shape[0])
    deg = [0] * nb
    nobst = [0] * nb
    for k in range(nc):
        deg[b1[k]] += 1
        if b2[k] < nb:
            deg[b2[k]] += 1
        else:
            nobst[b1[k]] += 1
    pinned = [False] * nb
    if e:
        An = np.asarray(A, dtype=np.float64).reshape(e, 3 * nb)
        for j in np.nonzero((An != 0).any(axis=0))[0]:
            pinned[int(j) // 3] = True
    border = [pinned[b] or deg[b] - nobst[b] > DEGB for b in range(nb)]
    rank = [0] * nb
    nbb = 0
    for b in range(nb):
        if border[b]:
            rank[b] = -1 - nbb
            nbb += 1
    nbd = 3 * nbb + e
    adj = [[] for _ in range(nb)]                           # entries 2 k + side, sorted by contact index
    for k in range(nc):
        adj[b1[k]].append(2 * k)
        if b2[k] < nb:
            adj[b2[k]].append(2 * k + 1)
    nbr = [[(b1[a >> 1] if a & 1 else b2[a >> 1]) for a in adj[b]] for b in range(nb)]
    nbr = [[o if o < nb else -1 for o in lst] for lst in nbr]
    mark = [-2 if border[b] else -1 for b in range(nb)]
    queue = [0] * nb
    px, py, comp = [0.0] * nb, [0.0] * nb, [0] * nb
    tail = ncomp = 0
    for root in range(nb):
        if mark[root] != -1:
            continue
        first = root
        for sweep in range(2):
            base = tail
            queue[base] = first
            mark[first] = base
            px[first] = py[first] = 0.0
            comp[first] = ncomp
            hd, tl, lvl_end = base, base + 1, base + 1
            while hd < tl:
                cnt = min(32, lvl_end - hd)
                lanes = queue[hd:hd + cnt]
                maxd = max(len(nbr[u]) for u in lanes)
                for k in range(maxd):
                    # every lane reads mark[] before any winner writes it; the lowest lane wins a shared body
                    seen = set()
                    wins = []
                    for u in lanes:
                        if k >= len(nbr[u]):
                            continue
                        w = nbr[u][k]
                        if w >= 0 and mark[w] == -1 and w not in seen:
                            seen.add(w)
                            wins.append((u, w))
                    for u, w in wins:
                        queue[tl] = w
                        mark[w] = tl
                        comp[w] = ncomp
                        ad = adj[u][k]
                        kc = ad >> 1
                        ddx = p1[kc][0] - p2[kc][0]
                        ddy = p1[kc][1] - p2[kc][1]
                        px[w] = px[u] - ddx if ad & 1 else px[u] + ddx
                        py[w] = py[u] - ddy if ad & 1 else py[u] + ddy
                        tl += 1
                hd += cnt
                if hd == lvl_end:
                    lvl_end = tl
            if sweep == 0:
                first = queue[tl - 1]
                for i in range(base, tl):
                    mark[queue[i]] = -1
            else:
                tail = tl
        ncomp += 1
    nband = tail
    band = [b for b in range(nb) if mark[b] >= 0]
    rkx, rky = [0] * nb, [0] * nb
    for r, b in enumerate(sorted(band, key=lambda b: (comp[b], px[b], b))):
        rkx[b] = r
    for r, b in enumerate(sorted(band, key=lambda b: (comp[b], py[b], b))):
        rky[b] = r
    widths = [0, 0, 0]
    for k in range(nc):
        u1, u2 = b1[k], b2[k]
        if u2 < nb and mark[u1] >= 0 and mark[u2] >= 0:
            widths[0] = max(widths[0], abs(mark[u1] - mark[u2]))
            widths[1] = max(widths[1], abs(rkx[u1] - rkx[u2]))
            widths[2] = max(widths[2], abs(rky[u1] - rky[u2]))
    choice, bwb = 0, widths[0]
    if widths[1] < bwb:
        choice, bwb = 1, widths[1]
    if widths[2] < bwb:
        choice, bwb = 2, widths[2]
    best = (mark, rkx, rky)[choice]
    for b in band:
        rank[b] = best[b]
    s = band_sizes(bwb)
    Nb = 3 * nband
    return dict(nband=nband, nbb=nbb, nbd=nbd, bwb=bwb, bw=s["bw"], bwa=s["bwa"], Nbp=(Nb + 7) & ~7,
                choice=choice, widths=tuple(widths), rank=rank)


def order_scene(sc):
    """`order` of a scene dict built below."""
    return order(sc["nb"], sc["body1"], sc["body2"], sc["p1"], sc["p2"], sc.get("A"))


# ------------------------------------------------------------------------------------------ scenes
def contacts_from_positions(pos, pairs, obstacle_pairs=(), floor_normal=(0.0, -1.0)):
    """Contact list of bodies at pos [nb, 2] (float64): a two-body contact per (i, j) in pairs at the midpoint,
    and a one-body contact per (i, depth) in obstacle_pairs against a static obstacle (body2 = nb) below."""
    pos = np.asarray(pos, dtype=np.float64)
    nb = pos.shape[0]
    b1, b2, nrm, p1, p2 = [], [], [], [], []
    for i, j in pairs:
        d = pos[i] - pos[j]
        dist = math.hypot(d[0], d[1])
        n = d / dist
        b1.append(i); b2.append(j); nrm.append(n); p1.append(-0.5 * dist * n); p2.append(0.5 * dist * n)
    for i, depth in obstacle_pairs:
        n = np.asarray(floor_normal, dtype=np.float64)
        b1.append(i); b2.append(nb); nrm.append(n); p1.append(-depth * n); p2.append(np.zeros(2))
    f = lambda a: np.asarray(a, dtype=np.float64).reshape(len(b1), 2)
    return dict(nb=nb, pos=pos, body1=np.asarray(b1, dtype=np.int32), body2=np.asarray(b2, dtype=np.int32),
                normal=f(nrm), p1=f(p1), p2=f(p2))


def lattice(W, H, families, spacing=2.0, tilt=1e-3):
    """W x H grid of bodies (body = y W + x); contacts join grid neighbours of the given (dx, dy) families in
    that order (scenes.pile_layout's families). `tilt` shears x by row so that no two bodies share an x (or y)
    coordinate: the x / y orderings have no ties."""
    pos = np.zeros((W * H, 2))
    for k in range(W * H):
        x, y = k % W, k // W
        pos[k] = (spacing * x + tilt * y, spacing * y + tilt * x)
    pairs = []
    for dx, dy in families:
        for k in range(W * H):
            x2, y2 = k % W + dx, k // W + dy
            if 0 <= x2 < W and 0 <= y2 < H:
                pairs.append((k, y2 * W + x2))
    return contacts_from_positions(pos, pairs)


FIVE = ((1, 0), (0, 1), (1, 1), (-1, 1), (2, 0))
SIX = FIVE + ((0, 2),)


def hex_pile(cols, rows, floor=True, pitch=2.0, tilt=1e-3):
    """Hexagonal pile `cols` wide and `rows` high (every touching neighbour a contact), resting on a floor body
    (body 0, pinned by 3 equality rows) that touches the whole bottom row: the shape of BASELINE config 4."""
    off = 1 if floor else 0
    nb = cols * rows + off
    pos = np.zeros((nb, 2))
    if floor:
        pos[0] = (pitch * cols / 2, 1.0e5)
    dy = pitch * math.sqrt(3) / 2
    idx = lambda r, c: off + r * cols + c
    for r in range(rows):
        for c in range(cols):
            pos[idx(r, c)] = (pitch * c + (r % 2) * pitch / 2 + tilt * r, -dy * r + tilt * c)
    pairs = []
    for r in range(rows):
        for c in range(cols):
            if c + 1 < cols:
                pairs.append((idx(r, c), idx(r, c + 1)))
            if r + 1 < rows:
                for c2 in ((c - 1, c) if r % 2 == 0 else (c, c + 1)):
                    if 0 <= c2 < cols:
                        pairs.append((idx(r, c), idx(r + 1, c2)))
    if floor:
        pairs += [(idx(0, c), 0) for c in range(cols)]
    sc = contacts_from_positions(pos, pairs)
    if floor:
        A = np.zeros((3, 3 * nb))
        A[0, 0] = A[1, 1] = A[2, 2] = 1.0
        sc["A"] = A
    return sc


def random_graph(nb, seed, max_deg=DEGB, mean_deg=6.0, extent=10.0):
    """Seeded random contact graph on nb bodies at random positions: about mean_deg contacts per body, none
    with more than max_deg; each pair at most once."""
    rng = np.random.default_rng(seed)
    pos = rng.uniform(0.0, extent, size=(nb, 2))
    deg = np.zeros(nb, dtype=int)
    pairs, seen = [], set()
    target = int(mean_deg * nb / 2)
    tries = 0
    while len(pairs) < target and tries < 50 * target:
        tries += 1
        i, j = (int(v) for v in rng.integers(0, nb, size=2))
        if i == j or (min(i, j), max(i, j)) in seen or deg[i] >= max_deg or deg[j] >= max_deg:
            continue
        seen.add((min(i, j), max(i, j)))
        deg[i] += 1; deg[j] += 1
        pairs.append((i, j))
    return contacts_from_positions(pos, pairs)


# Seeded random graphs at the band limits: (nb, seed, mean_deg) -> ordered half bandwidth (bodies).
# Found by scanning seeds with `order`; test_band_plan.py pins the widths.
WIDE_GRAPHS = {
    (42, 40, 12.0): 40,     # bwa = 128, the widest band the plan admits (n = 126: forced onto the banded kernel)
    (44, 17, 12.0): 42,     # Wc = 136 >= Nbp = 136: the window holds the whole matrix
    (45, 1, 12.0): 42,
    (50, 3, 8.0): 42,
    (58, 4, 6.0): 41,
    (50, 0, 12.0): 44,      # window A: bwa 136 > 128
    (58, 6, 8.0): 44,       # window A at its last body count
    (50, 5, 12.0): 45,      # bwa 144: past the window as well
}


def hubs(nhub, deg, ring=60, extent=40.0, obstacle_per_hub=0, seed=0, hub_links=()):
    """`nhub` hub bodies (0 .. nhub-1), each with `deg` two-body contacts to distinct bodies of a ring of `ring`
    bodies (which touch their ring neighbours), `obstacle_per_hub` one-body contacts each, and hub-hub contacts
    for the pairs in hub_links."""
    rng = np.random.default_rng(seed)
    nb = nhub + ring
    pos = np.zeros((nb, 2))
    for h in range(nhub):
        pos[h] = (extent * math.cos(2 * math.pi * h / max(nhub, 1)) * 0.3, extent * math.sin(2 * math.pi * h / max(nhub, 1)) * 0.3)
    for r in range(ring):
        a = 2 * math.pi * r / ring
        pos[nhub + r] = (extent * math.cos(a), extent * math.sin(a))
    pos += rng.uniform(-0.1, 0.1, size=pos.shape)
    pairs = [(nhub + r, nhub + (r + 1) % ring) for r in range(ring)]
    for h in range(nhub):
        for t in range(deg):
            pairs.append((h, nhub + (h * 7 + t * 3) % ring) if t % 2 == 0 else (nhub + (h * 7 + t * 3) % ring, h))
    pairs += list(hub_links)
    obst = [(h, 0.01) for h in range(nhub) for _ in range(obstacle_per_hub)]
    return contacts_from_positions(pos, pairs, obst)


def to_soa(sc, B=1, seed=0, vscale=1.0, mode=0):
    """Engine inputs for B copies of scene sc (float64 CPU tensors): the keys of scenes.make_contact_soa plus
    fext (gravity) and, when the scene has equality rows, A and b."""
    g = torch.Generator().manual_seed(seed)
    nb = sc["nb"]
    nc = len(sc["body1"])
    f64 = torch.float64
    mass = torch.rand(B, nb, generator=g, dtype=f64) + 0.5
    rad = torch.rand(B, nb, generator=g, dtype=f64) * 0.2 + 0.9
    rep = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(f64).unsqueeze(0).expand(B, *a.shape).contiguous()
    out = dict(mass=mass, inertia=0.5 * mass * rad * rad, v=torch.randn(B, 3 * nb, generator=g, dtype=f64) * vscale,
               normal=rep(sc["normal"]), p1=rep(sc["p1"]), p2=rep(sc["p2"]),
               mu=torch.rand(B, nc, generator=g, dtype=f64) * 0.8 + 0.1,
               restitution=torch.rand(B, nc, generator=g, dtype=f64) * 0.5 + 0.2,
               body1=torch.from_numpy(sc["body1"]).to(torch.int32), body2=torch.from_numpy(sc["body2"]).to(torch.int32))
    fext = torch.zeros(B, 3 * nb, dtype=f64)
    fext[:, 2::3] = 10.0 * mass
    out["fext"] = fext
    if "A" in sc:
        out["A"] = torch.from_numpy(sc["A"]).to(f64).unsqueeze(0).expand(B, -1, -1).contiguous()
        out["b"] = torch.zeros(B, sc["A"].shape[0], dtype=f64)
    return out
