"""GPU: the per-scene body walks at their limits -- the active contact walk (lcpb200_contacts_active,
csrc/lcp_contacts.cuh) and the tile walk SceneWalk (csrc/lcp_raycast.cuh) of lcpb200_raycast, lcpb200_signed_distance
and lcpb200_body_distance's nearest mode.

Both walks produce discrete outputs (pair lists, features, body indices), so everything here is compared exactly:
* the active walk, fp32 and fp64, against lcpb200_contacts on the standalone world of each scene's active bodies
  (bitwise: counts, lists mapped back, feat, geometry) and, on scenes of up to 1 100 bodies with few polygon pairs,
  against the float64 restatement tests/contact_ref.py with the tolerances of test_gpu_contact_limits.py: the
  compaction at nt = 1 024 / 1 025 / 8 191 / 8 192 (every word and warp boundary, nd at and around a multiple of 32
  and inside the last word), pair totals at the 1 024-pair chunk edges, 4.5 M pairs over 3 000 active bodies,
  degenerate activity and its padding, 2 (8 SMs) + 5 scenes per launch, per-scene masks with a padded stride, a
  capacity below the count, and a BatchedWorld of 1 100 circles against find_contacts_torch;
* SceneWalk, fp32 and fp64, against tests/ray_ref.py, tests/sdf_ref.py and tests/distance_ref.py: polygon tiles of
  every ptile class (256, 204, 7, 4 polygons) and circle tiles around 256, exact ties across tile boundaries and
  readings exactly at max_dist, activity at tile boundaries and at 8 192 bodies, 16 SMs + 7 scenes per launch with 33
  and 257 queries (bitwise equal to launches of at most 16 SMs items), and nearest mode with masks over tiles.
Every test first asserts that its scene crosses the limit it names, with the SM count read from the device.
"""
import math

import numpy as np
import pytest
import torch

from tests import contact_ref as cr
from tests.distance_ref import nearest_ref, pair_ref
from tests.test_gpu_contact_limits import F32_MARGIN, GEO, check_scene, coord_scale
from tests.test_gpu_distance import raw as dist_raw
from tests.test_gpu_hetero_world import active_walk, mask_words, sub_scene
from tests.test_gpu_raycast import raw as ray_raw, reference as ray_reference, scene as ray_scene
from tests.test_gpu_sdf import raw as sdf_raw, reference as sdf_reference

pytestmark = pytest.mark.gpu
f64, f32 = torch.float64, torch.float32
DTYPES = [f64, f32]

# ---------------------------------------------------------------------------------------------------- kernel constants
NT, ITEMS = 256, 4                  # lcp_contacts.cuh: threads per CTA, consecutive pairs per thread and chunk
CHUNK = NT * ITEMS                  # pairs per chunk of the contact walk
MAX_ACTIVE_NT = 8192                # bodies of a world walked per scene (32 bodies per thread)
TC, TV, TP = 256, 1024, 256         # lcp_raycast.cuh: circles, polygon vertices and polygons per tile


def ptile(nv):
    """polygons per SceneWalk tile"""
    return min(TV // nv, TP)


def launch_shape(B, n, sms):
    """(threads, chunks, grid) of a ray, point or body-distance launch of n queries in each of B scenes"""
    nth = NT if n >= NT else (n + 31) // 32 * 32
    chunks = (n + nth - 1) // nth
    return nth, chunks, min(B * chunks, 16 * sms)


def contact_grid(B, sms):
    return min(B, 8 * sms)


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def words_of(nt):
    return (nt + 31) // 32


# ---------------------------------------------------------------------------------------------------- A: scenes
def boxes(g, B, n, spread, w0, h0):
    """n rotated boxes per scene [B, n, 6, 2] (positive area, padded to 6 by repeating the last vertex)"""
    r = lambda *s: torch.rand(*s, generator=g, dtype=f64)
    c = spread * r(B, n, 1, 2)
    a = 2 * math.pi * r(B, n, 1)
    w, h = w0 * (1 + r(B, n, 1)), h0 * (1 + r(B, n, 1))
    lx = torch.tensor([0.5, 0.5, -0.5, -0.5], dtype=f64) * w
    ly = torch.tensor([-0.5, 0.5, 0.5, -0.5], dtype=f64) * h
    v = c + torch.stack([torch.cos(a) * lx - torch.sin(a) * ly, torch.sin(a) * lx + torch.cos(a) * ly], 3)
    return torch.cat([v, v[:, :, 3:].expand(B, n, 2, 2)], 2).contiguous()


def scenes(B, nb, npoly, no, spread, seed):
    """B random scenes of one shape in the layout of active_walk: circles of radius 4-10, boxes and obstacles"""
    g = torch.Generator().manual_seed(seed)
    pos = spread * torch.rand(B, nb, 2, generator=g, dtype=f64)
    rad = 4 + 6 * torch.rand(B, nb, generator=g, dtype=f64)
    pv = boxes(g, B, npoly, spread, 10.0, 6.0)
    ov = boxes(g, B, no, spread, 30.0, 8.0)
    pf = 0.2 + 0.6 * torch.rand(B, npoly, generator=g, dtype=f64)
    of = 0.2 + 0.6 * torch.rand(B, no, generator=g, dtype=f64)
    return [dict(pos=pos[s], rad=rad[s], polys=pv[s], obst=ov[s], pfric=pf[s], ofric=of[s]) for s in range(B)]


def ref_layout(sc):
    """a scene of active_walk's layout in the layout of tests/contact_ref.py, with active_walk's materials"""
    from lcp_physics_b200.world import polygon_centroid
    nb, npoly, no = sc["pos"].shape[0], sc["polys"].shape[0], sc["obst"].shape[0]
    cen = lambda v: polygon_centroid(v).numpy() if v.shape[0] else np.zeros((0, 2))
    return dict(pos=sc["pos"].numpy(), rad=sc["rad"].numpy(), fric=np.full(nb, 0.5), rest=np.zeros(nb),
                pverts=sc["polys"].numpy(), pcen=cen(sc["polys"]), pfric=sc["pfric"].numpy(), prest=np.zeros(npoly),
                overts=sc["obst"].numpy(), oref=cen(sc["obst"]), ofric=sc["ofric"].numpy(), orest=np.zeros(no))


def as_numpy(got):
    out = {k: got[k].cpu().numpy() for k in ("b1", "b2", "feat", "counts")}
    out.update({k: t.cpu().double().numpy() for k, t in zip(GEO, got["geo"])})
    return out


def standalone(got, s, sc, act, dtype, cap, excl=()):
    """scene s of an active-walk launch against lcpb200_contacts on the world of its active bodies alone: counts, the
    stored lists mapped back to body indices, feat and geometry bitwise. Returns (sub-world, index map, its pairs of
    excl)."""
    sub, idx = sub_scene(sc, act)
    inv = {int(k): q for q, k in enumerate(idx.tolist())}
    sub_excl = [(inv[a], inv[b]) for a, b in excl if a in inv and b in inv]
    n = int(got["counts"][s])
    if sub["pos"].shape[0] + sub["polys"].shape[0] == 0:                   # no dynamic body: no pair
        assert n == 0, s
        return sub, idx, sub_excl
    ref = active_walk([sub], dtype, cap, mask=mask_words(sub_excl, len(idx)) if sub_excl else None, plain=True)
    assert int(ref["counts"][0]) == n, (s, int(ref["counts"][0]), n)
    k = min(n, cap)
    m = idx.cuda()
    assert torch.equal(got["b1"][s, :k], m[ref["b1"][0, :k].long()].int()), s
    assert torch.equal(got["b2"][s, :k], m[ref["b2"][0, :k].long()].int()), s
    assert torch.equal(got["feat"][s, :k], ref["feat"][0, :k]), s
    for a, b in zip(got["geo"], ref["geo"]):
        assert torch.equal(a[s, :k], b[0, :k]), s
    return sub, idx, sub_excl


def against_restatement(out, s, sub, idx, sub_excl, dtype, cap, nb, nt, budget=2000):
    """scene s (as_numpy outputs) against contact_ref on its sub-world, indices mapped back, with the full world's
    padding; False when the sub-world is too large for the host restatement or (float32) a decision is too close to
    call"""
    nbs, nps, nos = sub["pos"].shape[0], sub["polys"].shape[0], sub["obst"].shape[0]
    if len(idx) > 1100 or nbs * (nps + nos) + nps * (nps - 1) // 2 + nps * nos > budget:
        return False
    if dtype == f32 and len(idx) > 200:            # larger scenes always hold a decision within float32 round-off
        return False
    rs = cr.rounded(ref_layout(sub), dtype)
    ref = cr.scene_contacts(rs, 0.1, cr.mask_words(len(idx), sub_excl) if sub_excl else None)
    if dtype == f32 and ref["margin"] <= F32_MARGIN * coord_scale(rs):
        return False
    m = idx.numpy()
    check_scene(out, s, dict(ref, b1=m[ref["b1"]], b2=m[ref["b2"]]), cap, nb, nt, dtype, coord_scale(rs), "mask")
    return True


# ---------------------------------------------------------------------------------------------------- A1: compaction
# (nb, np, no): nt = 1 024 (nd inside the last word), 1 025 (nd = 1 024, a multiple of 32), 8 191 (nd inside the last,
# partial word), 8 192 (nd one below and one above 8 160 = 255 x 32)
COMPACTION_SHAPES = [(1019, 2, 3), (1022, 2, 1), (8180, 2, 9), (8157, 2, 33), (8159, 2, 31)]
PATTERNS = ("all", "p10", "p60", "last_warp", "last_word", "gap_word")


def activity(name, nt, g):
    k = torch.arange(nt)
    word = k // 32
    W = words_of(nt)
    if name == "all":
        return torch.ones(nt, dtype=torch.bool)
    if name == "p10":
        return torch.rand(nt, generator=g) < 0.1
    if name == "p60":
        return torch.rand(nt, generator=g) < 0.6
    if name == "last_warp":                     # the words held by the last warp holding any (warp 7 at nt > 7 168)
        return word >= 32 * ((W - 1) // 32)
    if name == "last_word":
        return word == W - 1
    a = torch.rand(nt, generator=g) < 0.6     # gap_word: a fully inactive word between active ones
    a[word == W // 2] = False
    a[word == W // 2 - 1] = True
    a[word == W // 2 + 1] = True
    return a


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape", COMPACTION_SHAPES, ids=lambda s: "nt%d_nd%d" % (sum(s), s[0] + s[1]))
def test_compaction_at_word_and_warp_boundaries(shape, dtype):
    nb, npoly, no = shape
    nt, nd = sum(shape), nb + npoly
    W = words_of(nt)
    assert 1024 <= nt <= MAX_ACTIVE_NT and W >= 32                      # every lane of warp 0 holds a word
    assert nt == 1024 or W > 32                                        # beyond 1 024: words in a second warp
    assert nd % 32 in (0, 1, 31) or nd // 32 == W - 1                  # nd at a word boundary or in the last word
    g = torch.Generator().manual_seed(nt + nd)
    scs = scenes(len(PATTERNS), nb, npoly, no, 40.0 * math.sqrt(nt), seed=nt + nd)
    act = torch.stack([activity(p, nt, g) for p in PATTERNS])
    if nt == MAX_ACTIVE_NT:
        assert (W - 1) // 32 == NT // 32 - 1                           # all 256 threads hold a word, warp 7 too
    cap = nt
    got = active_walk(scs, dtype, cap, act)
    assert int(got["counts"].max()) > 0
    none = active_walk(scs[:1], dtype, cap)                             # all active == active NULL, bitwise
    for k in ("counts", "b1", "b2", "feat"):
        assert torch.equal(none[k][0], got[k][0]), k
    for a, b in zip(none["geo"], got["geo"]):
        assert torch.equal(a[0], b[0])
    out = as_numpy(got)
    checked = 0
    for s in range(len(PATTERNS)):
        sub, idx, sx = standalone(got, s, scs[s], act[s], dtype, cap)
        checked += against_restatement(out, s, sub, idx, sx, dtype, cap, nb, nt)
    assert checked >= (1 if dtype == f64 else 0), checked


# ---------------------------------------------------------------------------------------------------- A2: pair chunks
def chunk_world(B):
    """70 circles of radius 10 in a disc of radius 1 and 1 030 obstacles containing every centre: every pair of the
    walk is a contact"""
    sc = cr.all_contact_scene(70, 1030, nv=6, seed=4)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    one = dict(pos=t(sc["pos"]), rad=t(sc["rad"]), polys=torch.zeros(0, 6, 2, dtype=f64), obst=t(sc["overts"]),
               pfric=torch.zeros(0, dtype=f64), ofric=t(sc["ofric"]))
    return [one] * B


def chunk_totals():
    """(nd_s, no_s) of active lists whose pair totals sit at the 1 024-pair chunk edges: 1 023, 1 024, 1 025 and 2 049
    with active obstacles, 990 / 1 035 and 2 016 / 2 080 (45, 46, 64, 65 bodies) without"""
    out = [cr.shape_for_pairs(P, no_max=1030) for P in (1023, 1024, 1025, 2049)]
    return out + [(n, 0) for n in (45, 46, 64, 65)]


@pytest.mark.parametrize("dtype", DTYPES)
def test_pair_totals_at_chunk_edges(dtype):
    totals = chunk_totals()
    scs = chunk_world(len(totals))
    nb, no = 70, 1030
    nt = nb + no
    g = torch.Generator().manual_seed(2)
    act = torch.zeros(len(totals), nt, dtype=torch.bool)
    want = []
    for s, (nd_s, no_s) in enumerate(totals):
        assert nd_s <= nb and no_s <= no
        act[s, torch.randperm(nb, generator=g)[:nd_s]] = True
        act[s, nb + torch.randperm(no, generator=g)[:no_s]] = True
        want.append(cr.n_pairs(nd_s, 0, no_s))
    assert want[:4] == [1023, 1024, 1025, 2049] and {w // CHUNK for w in want} == {0, 1, 2}
    assert words_of(nt) > 32
    cap = 2100
    got = active_walk(scs, dtype, cap, act)
    for s in range(len(totals)):
        idx = act[s].nonzero()[:, 0].numpy()
        I, J = cr.pair_list(totals[s][0], 0, totals[s][1])
        assert int(got["counts"][s]) == want[s], s
        assert np.array_equal(got["b1"][s, :want[s]].cpu().numpy(), idx[I]), s
        assert np.array_equal(got["b2"][s, :want[s]].cpu().numpy(), idx[J]), s
        assert np.all(got["b1"][s, want[s]:].cpu().numpy() == 0) and np.all(got["b2"][s, want[s]:].cpu().numpy() == 1)
        standalone(got, s, scs[s], act[s], dtype, cap)


@pytest.mark.parametrize("dtype", DTYPES)
def test_three_thousand_active_bodies_contacts_in_first_and_last_chunk(dtype):
    """3 600 circles 10 apart (radius 1, no contact) and a far obstacle; 3 000 active: 4.5 M pairs in 4 393 chunks.
    The first two and the last two active bodies touch, and so does an inactive body placed on the first one."""
    nb, B = 3600, 2
    k = torch.arange(nb, dtype=f64)
    grid = torch.stack([10.0 * (k % 60), 10.0 * (k // 60)], 1)
    g = torch.Generator().manual_seed(3)
    act = torch.zeros(B, nb + 1, dtype=torch.bool)
    scs = []
    for s in range(B):
        act[s, torch.randperm(nb, generator=g)[:3000]] = True
        on = act[s].nonzero()[:, 0]
        pos = grid.clone()
        pos[on[1]] = pos[on[0]] + torch.tensor([1.5, 0.0], dtype=f64)
        pos[on[-1]] = pos[on[-2]] + torch.tensor([0.0, 1.0 + s], dtype=f64)
        off = (~act[s, :nb]).nonzero()[0, 0]
        pos[off] = pos[on[0]] - torch.tensor([1.0, 0.0], dtype=f64)   # touches an active body, but inactive
        scs.append(dict(pos=pos, rad=torch.ones(nb, dtype=f64), polys=torch.zeros(0, 6, 2, dtype=f64),
                        obst=boxes(g, 1, 1, 10.0, 5.0, 5.0)[0] - 500.0, pfric=torch.zeros(0, dtype=f64),
                        ofric=torch.full((1,), 0.5, dtype=f64)))
    npairs = cr.n_pairs(3000, 0, 0)
    assert npairs > 2_000_000 and (npairs - 1) // CHUNK > 4000
    cap = 8
    got = active_walk(scs, dtype, cap, act)
    out = as_numpy(got)
    for s in range(B):
        on = act[s].nonzero()[:, 0]
        assert int(got["counts"][s]) == 2
        assert got["b1"][s, :2].tolist() == [int(on[0]), int(on[-2])] and got["b2"][s, :2].tolist() == [int(on[1]), int(on[-1])]
        sub, idx, sx = standalone(got, s, scs[s], act[s], dtype, cap)
        rs = cr.rounded(ref_layout(sub), dtype)
        ref = cr.scene_contacts(rs, 0.1)
        m = idx.numpy()
        check_scene(out, s, dict(ref, b1=m[ref["b1"]], b2=m[ref["b2"]]), cap, nb, nb + 1, dtype, coord_scale(rs), "mask")


# ---------------------------------------------------------------------------------------------------- A3: degenerate
def degenerate_worlds():
    """(scene, activity rows): 40 circles of radius 10 around the origin with 2 boxes and 3 obstacles around them
    (every pair a contact), and a world without circles (the boxes of contact_ref.aligned_stack)"""
    a = cr.all_contact_scene(40, 3, nv=6, seed=6)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x))
    polys = np.stack([cr.box(-3, -3, 3, 3, 6), cr.box(-2, -4, 4, 2, 6)])
    circ = dict(pos=t(a["pos"]), rad=t(a["rad"]), polys=t(polys), obst=t(a["overts"]),
                pfric=torch.full((2,), 0.4, dtype=f64), ofric=t(a["ofric"]))
    nt = 45
    rows = []
    for on in ([], [5], [5, 9], [42, 43, 44], [7, 42, 43, 44], [40, 42, 43], [2, 3, 4, 40, 41, 44], list(range(nt))):
        r = torch.zeros(nt, dtype=torch.bool)
        r[on] = True
        rows.append(r)
    st = cr.aligned_stack(6)
    np_, no = st["pverts"].shape[0], st["overts"].shape[0]
    poly = dict(pos=torch.zeros(0, 2, dtype=f64), rad=torch.zeros(0, dtype=f64), polys=t(st["pverts"]),
                obst=t(st["overts"]), pfric=t(st["pfric"]), ofric=t(st["ofric"]))
    prows = []
    for on in ([], [3], [np_, np_ + 1], [0, np_], list(range(2, np_ + no))):
        r = torch.zeros(np_ + no, dtype=torch.bool)
        r[on] = True
        prows.append(r)
    return [(circ, torch.stack(rows)), (poly, torch.stack(prows))]


@pytest.mark.parametrize("dtype", DTYPES)
def test_degenerate_activity_and_padding(dtype):
    """0, 1 and 2 active bodies, only obstacles, one dynamic body with obstacles, bodies 0 and 1 inactive: counts,
    lists and what the walk writes past them (the padding pair (0, 1) of the full body list, feat -1 or 0 without
    circles, penetration -1e30) as contact_ref.truncate defines it"""
    for sc, act in degenerate_worlds():
        nb, npoly, no = sc["pos"].shape[0], sc["polys"].shape[0], sc["obst"].shape[0]
        nt = nb + npoly + no
        assert bool((act.sum(1) <= 2).any()) and bool((~act[:, :2]).all(1).any())
        B = act.shape[0]
        for cap in (6, 64):
            got = active_walk([sc] * B, dtype, cap, act)
            out = as_numpy(got)
            for s in range(B):
                sub, idx, sx = standalone(got, s, sc, act[s], dtype, cap)
                assert against_restatement(out, s, sub, idx, sx, dtype, cap, nb, nt) or dtype == f32, s
            counts = got["counts"].tolist()
            assert 0 in counts and max(counts) > cap or cap == 64


# ---------------------------------------------------------------------------------------------------- A4: scenes/CTA
@pytest.mark.parametrize("dtype", DTYPES)
def test_several_scenes_per_cta(dtype):
    """B = 2 (8 SMs) + 5: CTA c walks scenes c, c + 8 SMs (and c + 16 SMs); an all-inactive scene directly before
    a busy one (odd c), a busy one before a one-body scene (even c), random activity in the third round"""
    sms = num_sms()
    grid = 8 * sms
    B = 2 * grid + 5
    assert contact_grid(B, sms) == grid and B > 2 * grid
    nb, npoly, no = 60, 2, 2
    nt = nb + npoly + no
    scs = scenes(B, nb, npoly, no, 100.0, seed=8)
    g = torch.Generator().manual_seed(8)
    act = torch.zeros(B, nt, dtype=torch.bool)
    for s in range(B):
        c, r = s % grid, s // grid
        if r == 0:
            act[s] = c % 2 == 0                                       # busy, or nothing active
        elif r == 1:
            if c % 2:
                act[s] = True
            else:
                act[s, c % nb] = True                                 # one body
        else:
            act[s] = torch.rand(nt, generator=g) < 0.2 + 0.15 * c
    cap = 96
    got = active_walk(scs, dtype, cap, act)
    for a in range(0, B, grid):                                       # at most 8 SMs scenes per launch
        part = active_walk(scs[a:a + grid], dtype, cap, act[a:a + grid])
        for k in ("counts", "b1", "b2", "feat"):
            assert torch.equal(part[k], got[k][a:a + grid]), (a, k)
        for x, y in zip(part["geo"], got["geo"]):
            assert torch.equal(x, y[a:a + grid]), a
    sample = sorted({0, 1, 2, 3, grid - 1, grid, grid + 1, grid + 2, 2 * grid - 1} | set(range(5, 2 * grid, grid // 4))
                    | set(range(B - 5, B)))
    assert len(sample) >= 16
    out = as_numpy(got)
    checked = 0
    for s in sample:
        sub, idx, sx = standalone(got, s, scs[s], act[s], dtype, cap)
        checked += against_restatement(out, s, sub, idx, sx, dtype, cap, nb, nt)
    assert checked >= (len(sample) if dtype == f64 else 1), checked
    counts = got["counts"]
    assert int(counts[1]) == 0 and int(counts[grid + 1]) > 0 and int(counts[grid]) == 0 and int(counts[0]) > 0


# ---------------------------------------------------------------------------------------------------- A5: masks
def bit31_pairs(sc, on, nt, count, g):
    """moves `count` active circles j onto active circles i with (i nt + j) % 32 == 31 (bit 31 of its mask word)"""
    pairs = []
    circles = [int(k) for k in on if k < sc["pos"].shape[0]]
    used = set()
    for i in circles:
        if len(pairs) == count:
            break
        j = next((j for j in circles if j > i and (i * nt + j) % 32 == 31 and j not in used and i not in used), None)
        if j is None:
            continue
        sc["pos"][j] = sc["pos"][i] + torch.tensor([1.0, 0.5], dtype=f64)
        used |= {i, j}
        pairs.append((i, j))
    assert len(pairs) == count
    return pairs


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("stride", ["padded", "shared", "none"])
def test_per_scene_masks(stride, dtype):
    """nc_stride = mask words + 13 with all-ones gaps (a wrong stride excludes pairs it should not), stride 0 (one
    mask) and no mask; excluded contacts on bit 31 and excluded pairs with an inactive body"""
    nb, npoly, no, B = 1060, 1, 1, 3
    nt = nb + npoly + no
    W = (nt * nt + 31) // 32
    assert words_of(nt) > 32
    scs = scenes(B, nb, npoly, no, 40.0 * math.sqrt(nt), seed=9)
    g = torch.Generator().manual_seed(9)
    act = torch.rand(B, nt, generator=g) < 0.8
    excl = []
    for s in range(B):
        on = act[s].nonzero()[:, 0].tolist()
        b31 = bit31_pairs(scs[s], on, nt, 3, g)
        off = (~act[s]).nonzero()[:, 0].tolist()
        excl.append(b31 + [(min(a, b), max(a, b)) for a, b in zip(off[:20], on[5:25]) if a != b])
    free = active_walk(scs, dtype, 2048, act)
    for s in range(B):                                                 # and a third of each scene's contacts
        n = int(free["counts"][s])
        pr = sorted({(int(a), int(b)) for a, b in zip(free["b1"][s, :n].tolist(), free["b2"][s, :n].tolist())})
        excl[s] += [p for p in pr[::3] if p not in excl[s]]
    if stride == "padded":
        words = torch.stack([mask_words(e, nt) for e in excl])
        mk = torch.full((B, W + 13), -1, dtype=torch.int32)
        mk[:, :W] = words
        got = active_walk(scs, dtype, 2048, act, mk, W + 13)
        per = excl
    elif stride == "shared":
        got = active_walk(scs, dtype, 2048, act, mask_words(excl[0], nt), 0)
        per = [excl[0]] * B
    else:
        got = active_walk(scs, dtype, 2048, act)
        per = [[]] * B
    out = as_numpy(got)
    checked = 0
    for s in range(B):
        sub, idx, sx = standalone(got, s, scs[s], act[s], dtype, 2048, per[s])
        checked += against_restatement(out, s, sub, idx, sx, dtype, 2048, nb, nt)
        n = int(got["counts"][s])
        pairs = set(zip(got["b1"][s, :n].tolist(), got["b2"][s, :n].tolist()))
        assert not pairs & set(per[s])
        if stride == "padded" or (stride == "shared" and s == 0):
            assert n < int(free["counts"][s]), s                       # the mask excluded contacts
        if stride == "none":
            assert n == int(free["counts"][s]), s
    assert checked >= (B if dtype == f64 else 0), checked


# ---------------------------------------------------------------------------------------------------- A6: capacity
@pytest.mark.parametrize("dtype", DTYPES)
def test_capacity_below_the_count(dtype):
    nb, npoly, no, B = 2000, 3, 2, 2
    nt = nb + npoly + no
    scs = scenes(B, nb, npoly, no, 20.0 * math.sqrt(nt), seed=10)
    act = torch.rand(B, nt, generator=torch.Generator().manual_seed(10)) < 0.9
    full = active_walk(scs, dtype, 8192, act)
    counts = full["counts"]
    assert int(counts.min()) > 2 * CHUNK // ITEMS and int(counts.max()) < 8192
    for s in range(B):
        standalone(full, s, scs[s], act[s], dtype, 8192)
    for cap in (1, int(counts.min()) // 3, int(counts.min()) - 1):
        got = active_walk(scs, dtype, cap, act)
        assert torch.equal(got["counts"], counts), cap                  # the true count
        for k in ("b1", "b2", "feat"):
            assert torch.equal(got[k], full[k][:, :cap]), (cap, k)
        for a, b in zip(got["geo"], full["geo"]):
            assert torch.equal(a, b[:, :cap]), cap


# ---------------------------------------------------------------------------------------------------- A7: BatchedWorld
def test_batched_world_of_1100_circles_matches_find_contacts_torch():
    """1 100 circles on a grid whose neighbours touch, a floor and a wall, per-scene activity and no_contact"""
    from lcp_physics_b200.world import BatchedWorld, rect_vertices
    B, nb = 3, 1100
    k = torch.arange(nb, dtype=f64)
    pos = torch.stack([9.5 * (k % 50), 9.5 * (k // 50)], 1).expand(B, -1, -1).contiguous()
    obst = torch.stack([rect_vertices([230.0, -10.0], [500.0, 10.0]), rect_vertices([-10.0, 100.0], [10.0, 230.0])])
    nt = nb + 2
    assert words_of(nt) > 32 and nb > CHUNK
    g = torch.Generator().manual_seed(11)
    act = torch.rand(B, nt, generator=g) < 0.7
    act[:, nb:] = True
    excl = [[(i, i + 1) for i in range(s, nb - 1, 5)] + [(i, i + 50) for i in range(0, nb - 50, 9)] + [(3, nb)]
            for s in range(B)]
    w = BatchedWorld(pos, 5.0, obstacles=obst, active=act, no_contact=excl, contact_capacity=4096,
                     strict_no_penetration=False, device="cuda")
    assert w.per_scene and w.nc_stride > 0
    w.find_contacts()
    counts, b1, b2 = w.find_contacts_torch()
    assert torch.equal(counts, w.counts) and int(counts.min()) > 500
    for s in range(B):
        n = int(counts[s])
        assert torch.equal(b1[s, :n], w.c_b1[s, :n]) and torch.equal(b2[s, :n], w.c_b2[s, :n]), s
        assert not set(zip(w.c_b1[s, :n].tolist(), w.c_b2[s, :n].tolist())) & set(excl[s])


# ---------------------------------------------------------------------------------------------------- B: scenes
def query_scene(B, nb, np_, no, V, n, seed, L=100.0):
    """ray scene of test_gpu_raycast (n rays per scene) with n query points"""
    sc = ray_scene(B, nb, np_, no, V, n, seed, L=L)
    g = torch.Generator().manual_seed(seed + 1)
    sc["x"] = (L + 20) * torch.rand(B, n, 2, generator=g, dtype=f64) - 10
    return sc


def nt_of(sc):
    return sc["pos"].shape[1] + sum(0 if sc[k] is None else sc[k].shape[1] for k in ("pv", "ov"))


def check_rays(sc, dtype, md, active=None):
    t, body, feat, n = ray_raw(sc, dtype, md, active)
    rt, rb, rf, rn, m = ray_reference(sc, dtype, md, active)
    ok = m > (1e-9 if dtype == f64 else 1e-3)
    assert float(ok.float().mean()) > 0.5, float(ok.float().mean())
    assert torch.equal(body[ok], rb[ok]) and torch.equal(feat[ok], rf[ok])
    tol, tol_n, floor = (1e-12, 1e-10, 1.0) if dtype == f64 else (1e-4, 1e-3, 10.0)
    assert float(((t.double() - rt).abs() / rt.abs().clamp_min(floor))[ok].max()) <= tol
    assert float((n.double() - rn).abs()[ok].max()) <= tol_n
    return body


def check_points(sc, dtype, md, active=None):
    s, body, feat, n = sdf_raw(sc, dtype, md, active)
    rs, rb, rf, rn, m = sdf_reference(sc, dtype, md, active)
    ok = m > (1e-9 if dtype == f64 else 1e-3)
    assert float(ok.float().mean()) > 0.5, float(ok.float().mean())
    assert torch.equal(body[ok], rb[ok]) and torch.equal(feat[ok], rf[ok])
    tol, tol_n, floor = (1e-12, 1e-10, 1.0) if dtype == f64 else (1e-4, 1e-3, 10.0)
    assert float(((s.double() - rs).abs() / rs.abs().clamp_min(floor))[ok].max()) <= tol
    # (x - q) / |x - q| next to a polygon's surface loses |x| eps / |x - q| to cancellation: compared where that stays
    # below 1e-4 (|sdf| > 1e-3 in fp64, as test_gpu_sdf.py, and > 0.1 in fp32)
    nm = ok & (rs.abs() > (1e-3 if dtype == f64 else 0.1))
    assert not bool(nm.any()) or float((n.double() - rn).abs()[nm].max()) <= tol_n
    return body


def rounded(sc, dtype):
    return {k: (None if sc[k] is None else sc[k].to(dtype).double()) for k in ("pos", "rad", "pv", "ov")}


def check_nearest(sc, dtype, md, q, active=None, nc=None, stride=0, excluded=None):
    """nearest mode for query bodies q [B, K] against nearest_ref on the scene rounded to dtype"""
    d, body, feat, n, pa = dist_raw(sc, dtype, md, q, active=active, nc=nc, nc_stride=stride)
    r = rounded(sc, dtype)
    rd, rb, rn, rm = nearest_ref(r["pos"], r["rad"], r["pv"], r["ov"], q, md, active, excluded)
    robust, tol = (1e-9, 1e-12) if dtype == f64 else (1e-3, 1e-4)
    scale = rd.abs().clamp_min(1.0)
    ok = rm > robust * scale
    assert bool(ok.any())
    body, d = body.cpu(), d.cpu().double()
    assert torch.equal(body[ok], rb[ok])
    far = (rd - md).abs() > robust * scale
    assert not bool((ok & far).any()) or float(((d - rd).abs() / scale)[ok & far].max()) <= tol
    return body


def nearest_queries(sc, B):
    """up to 12 circles and 2 polygons of the scene as nearest-mode queries [B, K]"""
    nb, nt = sc["pos"].shape[1], nt_of(sc)
    q = list(range(0, nb, max(1, nb // 12)))[:12] + list(range(nb, nt, max(1, (nt - nb) // 2)))[:2]
    return torch.tensor(q).expand(B, -1).contiguous()


def check_all(sc, dtype, md, active=None):
    B = sc["pos"].shape[0]
    check_rays(sc, dtype, md, active)
    check_points(sc, dtype, md, active)
    check_nearest(sc, dtype, md, nearest_queries(sc, B), active)


# ---------------------------------------------------------------------------------------------------- B1: tiles
# (nb, np, no, nv, L): polygons around every ptile class, circles around TC, no circles, circles only, one body. The
# dense polygon cases keep coordinates within 110, the scale the float32 tolerances of check_rays / check_points were
# set for (an fp32 edge normal carries the vertices' round-off over the edge length)
TILE_CASES = [
    (20, 200, 56, 3, 100.0), (20, 200, 57, 3, 100.0), (20, 400, 113, 3, 100.0),
    (20, 200, 56, 4, 100.0), (20, 200, 57, 4, 100.0), (20, 400, 113, 4, 100.0),
    (20, 180, 25, 5, 100.0), (20, 380, 29, 5, 100.0),
    (10, 5, 3, 129, 80.0), (10, 3, 2, 256, 80.0), (10, 6, 3, 256, 80.0),
    (255, 2, 1, 6, 150.0), (256, 2, 1, 6, 150.0), (257, 2, 1, 6, 150.0), (513, 2, 1, 6, 200.0),
    (0, 300, 2, 4, 250.0), (300, 0, 0, 0, 150.0), (1, 0, 0, 0, 20.0), (0, 1, 0, 5, 20.0),
]


def tile_id(c):
    nb, np_, no, nv, _ = c
    return "nb%d_npo%d_nv%d" % (nb, np_ + no, nv)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", TILE_CASES, ids=tile_id)
def test_tiles_of_every_size(case, dtype):
    nb, np_, no, nv, L = case
    npo = np_ + no
    # each case sits at or past a tile of polygons or of circles, or is a world without one of the two groups
    assert nb == 0 or npo == 0 or npo >= ptile(nv) or nb >= TC - 1
    sc = query_scene(2, nb, np_, no, nv, 300, seed=nb * 7 + npo * 3 + nv, L=L)
    md = 2.0 * L
    if nb + npo == 1:                                                   # one body: rays and points aimed at it
        g = torch.Generator().manual_seed(1)
        c = sc["pos"][:, :1] if nb else sc["pv"][:, :1].mean(2)
        a = 2 * math.pi * torch.rand(2, 300, generator=g, dtype=f64)
        sc["o"] = c - 15 * torch.stack([torch.cos(a), torch.sin(a)], 2)
        sc["u"] = (c + torch.rand(2, 300, 2, generator=g, dtype=f64) - 0.5 - sc["o"])
        sc["u"] = sc["u"] / sc["u"].norm(dim=2, keepdim=True)
        sc["x"] = c + 20 * (torch.rand(2, 300, 2, generator=g, dtype=f64) - 0.5)
    body = check_rays(sc, dtype, md)
    assert float((body >= 0).float().mean()) > 0.05
    check_points(sc, dtype, md)
    if nb + npo > 1:
        check_nearest(sc, dtype, md, nearest_queries(sc, 2))


# ---------------------------------------------------------------------------------------------------- B2: ties
def tie_scene():
    """300 circles and 210 + 10 pentagons (ptile 204) in [0, 100]^2, and isolated bit-identical duplicates: circles 10
    and 266 (= 10 + TC), 20 and 21 (one tile); polygons 3 and 207 (= 3 + ptile), polygon 10 and obstacle 214, polygons
    30 and 31; each pair with a probe circle (40 + k) 6 to its right. Returns the scene and [(lower, higher, centre)]."""
    nb, np_, no, nv = 300, 210, 10, 5
    sc = query_scene(1, nb, np_, no, nv, 64, seed=77)
    dups = []
    for k, (a, b) in enumerate([(10, 266), (20, 21)]):
        c = torch.tensor([300.0, 40.0 * k], dtype=f64)
        sc["pos"][0, a] = sc["pos"][0, b] = c
        sc["rad"][0, a] = sc["rad"][0, b] = 2.5
        dups.append((a, b, c))
    P = lambda q: (sc["pv"], q) if q < np_ else (sc["ov"], q - np_)
    pent = lambda c: c + 3.0 * torch.stack([torch.cos(torch.arange(5, dtype=f64) * 2 * math.pi / 5 + 0.3),
                                            torch.sin(torch.arange(5, dtype=f64) * 2 * math.pi / 5 + 0.3)], 1)
    for k, (qa, qb) in enumerate([(3, 207), (10, 214), (30, 31)]):
        c = torch.tensor([300.0, 80.0 + 40.0 * k], dtype=f64)
        v = pent(c)
        for q in (qa, qb):
            t, i = P(q)
            t[0, i] = v
        dups.append((nb + qa, nb + qb, c))
    for k, (_, _, c) in enumerate(dups):
        sc["pos"][0, 40 + k] = c + torch.tensor([6.0, 0.0], dtype=f64)
        sc["rad"][0, 40 + k] = 0.5
    # rays from 20 to the left of each pair, straight and at +-0.05 rad; points left of, above and at each centre
    o, u, x = [], [], []
    for _, _, c in dups:
        for ang in (-0.05, 0.0, 0.05):
            o.append(c - torch.tensor([20.0, 0.0], dtype=f64) + torch.tensor([0.0, 0.3], dtype=f64))
            u.append(torch.tensor([math.cos(ang), math.sin(ang)], dtype=f64))
        x += [c + torch.tensor([-0.2, 4.0], dtype=f64), c + torch.tensor([0.0, -4.5], dtype=f64),
              c + torch.tensor([0.1, 0.2], dtype=f64)]
    sc["o"], sc["u"], sc["x"] = torch.stack(o)[None], torch.stack(u)[None], torch.stack(x)[None]
    return sc, dups


@pytest.mark.parametrize("dtype", DTYPES)
def test_exact_ties_across_tile_boundaries_go_to_the_lower_index(dtype):
    sc, dups = tie_scene()
    nb, nt = sc["pos"].shape[1], nt_of(sc)
    pt = ptile(5)
    assert pt == 204 and TV % 5 != 0
    assert (10 // TC, 266 // TC) == (0, 1) and (3 // pt, 207 // pt) == (0, 1) and (10 // pt, 214 // pt) == (0, 1)
    assert 214 >= sc["pv"].shape[1]                                      # an obstacle duplicating a dynamic polygon
    md = 1000.0
    q = torch.tensor([[40 + k for k in range(len(dups))]])
    ones = torch.ones(1, nt, dtype=torch.bool)
    hi_off, lo_off = ones.clone(), ones.clone()
    for a, b, _ in dups:
        hi_off[0, b] = False
        lo_off[0, a] = False

    def run(active):
        return (ray_raw(sc, dtype, md, active), sdf_raw(sc, dtype, md, active),
                dist_raw(sc, dtype, md, q, active=active))

    base, alone, other = run(None), run(hi_off), run(lo_off)
    lower = torch.tensor([a for a, _, _ in dups])
    higher = torch.tensor([b for _, b, _ in dups])
    for k, (x, y) in enumerate(zip(base, alone)):                      # bitwise the scene without the duplicates
        for a, b in zip(x, y):
            assert torch.equal(a, b), k
    # every query hits its pair: rays and points three per pair, distance queries one
    assert torch.equal(base[0][1][0].cpu(), lower.repeat_interleave(3))
    assert torch.equal(base[1][1][0].cpu(), lower.repeat_interleave(3))
    assert torch.equal(base[2][1][0].cpu(), lower)
    # the higher duplicate alone is read at its own index with the same values
    assert torch.equal(other[0][1][0].cpu(), higher.repeat_interleave(3))
    assert torch.equal(other[1][1][0].cpu(), higher.repeat_interleave(3))
    assert torch.equal(other[2][1][0].cpu(), higher)
    for k in range(3):
        for i, (a, b) in enumerate(zip(other[k], base[k])):
            assert i == 1 or torch.equal(a, b), (k, i)


@pytest.mark.parametrize("dtype", DTYPES)
def test_readings_exactly_at_max_dist(dtype):
    """integer geometry: a ray entering a circle and one entering a box at t = 8, points at sdf 8, two circles 8
    apart; with max_dist = 8 each is read (the first hit is inclusive), and a copy of each body further down the list
    at the same reading is not"""
    box = lambda x0, y0, x1, y1: torch.tensor([[x0, y0], [x1, y0], [x1, y1], [x0, y1]], dtype=f64)
    pos = torch.tensor([[[0.0, 0.0], [12.0, 0.0], [0.0, 0.0]]])              # circle 2 duplicates circle 0
    rad = torch.full((1, 3), 2.0, dtype=f64)
    pv = torch.stack([box(8, 19, 12, 21), box(8, 19, 12, 21)])[None]         # polygon 4 duplicates polygon 3
    sc = dict(pos=pos, rad=rad, pv=pv, ov=None,
              o=torch.tensor([[[-10.0, 0.0], [0.0, 20.0]]]), u=torch.tensor([[[1.0, 0.0], [1.0, 0.0]]]),
              x=torch.tensor([[[-10.0, 0.0], [0.0, 20.0]]]))
    t, body, _, _ = ray_raw(sc, dtype, 8.0)
    assert t.tolist() == [[8.0, 8.0]] and body.tolist() == [[0, 3]]
    s, body, _, _ = sdf_raw(sc, dtype, 8.0)
    assert s.tolist() == [[8.0, 8.0]] and body.tolist() == [[0, 3]]
    d, body, _, _, _ = dist_raw(sc, dtype, 8.0, torch.tensor([[1]]))
    assert d.tolist() == [[8.0]] and body.tolist() == [[0]]
    t, body, _, _ = ray_raw(sc, dtype, 7.75)                                  # just short of it: no hit
    assert t.tolist() == [[7.75, 7.75]] and body.tolist() == [[-1, -1]]


# ---------------------------------------------------------------------------------------------------- B3: activity
@pytest.mark.parametrize("dtype", DTYPES)
def test_activity_at_tile_boundaries(dtype):
    """the first and last circle and polygon of a tile inactive, and a whole polygon tile inactive"""
    nb, np_, no, nv = 520, 400, 120, 4
    sc = query_scene(2, nb, np_, no, nv, 300, seed=33, L=300.0)
    nt = nb + np_ + no
    pt = ptile(nv)
    assert nb > 2 * TC and np_ + no > 2 * pt
    g = torch.Generator().manual_seed(34)
    act = torch.rand(2, nt, generator=g) < 0.8
    for b in (0, TC - 1, TC, 2 * TC - 1, 2 * TC):
        act[:, b] = False
    for q in (0, pt - 1, 2 * pt):
        act[:, nb + q] = False
    act[0, nb + pt:nb + 2 * pt] = False                                  # a whole tile
    act[1, nb + 2 * pt - 1] = False
    check_all(sc, dtype, 600.0, act)


@pytest.mark.parametrize("dtype", DTYPES)
def test_largest_world_with_active(dtype):
    nb, np_, no, nv = 7900, 200, 92, 6
    nt = nb + np_ + no
    assert nt == MAX_ACTIVE_NT and nb > 30 * TC and np_ + no > ptile(nv)
    sc = query_scene(1, nb, np_, no, nv, 300, seed=35, L=900.0)
    act = torch.rand(1, nt, generator=torch.Generator().manual_seed(36)) < 0.6
    check_all(sc, dtype, 300.0, act)


# ---------------------------------------------------------------------------------------------------- B4: items/CTA
def split_equal(fn, sc, per, B, *args):
    """fn on the whole batch equals fn on consecutive slices of `per` scenes, bitwise"""
    full = fn(sc, *args)
    for a in range(0, B, per):
        part = fn({k: (v[a:a + per] if isinstance(v, torch.Tensor) else v) for k, v in sc.items()}, *args)
        for x, y in zip(full, part):
            if x is not None:
                assert torch.equal(x[a:a + per], y), a
    return full


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n", [33, 257])
def test_several_items_per_cta(n, dtype):
    sms = num_sms()
    B = 16 * sms + 7
    nth, chunks, grid = launch_shape(B, n, sms)
    assert B * chunks > grid == 16 * sms
    assert (nth, chunks) == ((64, 1) if n == 33 else (256, 2))        # 31 dead lanes; one live thread in chunk 2
    sc = query_scene(B, 20, 6, 4, 6, n, seed=n, L=60.0)
    nt = 30
    per = grid // chunks                                                # at most 16 SMs items per launch
    md = 40.0
    rays = split_equal(lambda s: ray_raw(s, dtype, md), sc, per, B)
    pts = split_equal(lambda s: sdf_raw(s, dtype, md), sc, per, B)
    g = torch.Generator().manual_seed(n)
    a = torch.randint(0, nt, (B, n), generator=g)
    pairs = torch.stack([a, (a + torch.randint(1, nt, (B, n), generator=g)) % nt], 2)
    sc["ba"], sc["bb"] = pairs[..., 0], pairs[..., 1]
    dist = lambda s, near: dist_raw(s, dtype, md, s["ba"], None if near else s["bb"])
    pair_out = split_equal(dist, sc, per, B, False)
    near_out = split_equal(dist, sc, per, B, True)
    for near, full in ((False, pair_out), (True, near_out)):             # shared queries = expanded ones
        sh = dist_raw(sc, dtype, md, pairs[0, :, 0], None if near else pairs[0, :, 1], shared=True)
        ex = dist_raw(sc, dtype, md, pairs[0, :, 0].expand(B, n), None if near else pairs[0, :, 1].expand(B, n))
        for x, y in zip(sh, ex):
            assert torch.equal(x, y)
    sample = sorted({0, 1, per - 1, per, grid - 1, grid, B // 2} | set(range(B - 5, B)))
    sub = {k: (v[sample] if isinstance(v, torch.Tensor) else v) for k, v in sc.items()}
    assert torch.equal(check_rays(sub, dtype, md), rays[1][sample])
    assert torch.equal(check_points(sub, dtype, md), pts[1][sample])
    r = rounded(sub, dtype)
    k = min(n, 33)
    qp = pairs[sample][:, :k]
    rd, rhit, _, rm = pair_ref(r["pos"], r["rad"], r["pv"], r["ov"], qp, md)
    robust, tol = (1e-9, 1e-12) if dtype == f64 else (1e-3, 1e-4)
    scale = rd.abs().clamp_min(1.0)
    ok = rm > robust * scale
    got_d, got_b = pair_out[0][sample][:, :k].cpu().double(), pair_out[1][sample][:, :k].cpu()
    assert float(ok.double().mean()) > 0.5
    assert torch.equal(got_b[ok], torch.where(rhit, qp[..., 1], -1)[ok])
    far = (rd - md).abs() > robust * scale
    assert not bool((ok & far).any()) or float(((got_d - rd).abs() / scale)[ok & far].max()) <= tol
    q = pairs[sample][:, :k, 0]
    nd, nbody, _, _, _ = dist_raw(sub, dtype, md, q)
    assert torch.equal(nbody, near_out[1][sample][:, :k])
    check_nearest(sub, dtype, md, q)


# ---------------------------------------------------------------------------------------------------- B5: masks
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("stride", ["padded", "shared"])
def test_nearest_masks_across_tiles(stride, dtype):
    """per-scene no_contact with nc_stride = mask words + 13 (all-ones gaps), or one mask (stride 0), excluding each
    query's unmasked nearest body, candidates on both sides of the circle tile boundary (255 | 256) and of the
    polygon tile boundary (ptile(129) = 7), and pairs on bit 31 of a word"""
    from lcp_physics_b200.world import no_contact_masks
    B, nb, np_, no, nv = 3, 300, 5, 4, 129
    nt = nb + np_ + no
    pt = ptile(nv)
    assert pt == 7 and np_ + no > pt and nb > TC
    sc = query_scene(B, nb, np_, no, nv, 32, seed=41, L=60.0)
    q = torch.tensor(list(range(250, 262)) + list(range(nb, nt)) + [0, 1]).expand(B, -1).contiguous()
    md = 100.0
    free = dist_raw(sc, dtype, md, q)[1].cpu()
    per = []
    for s in range(B):
        ex = set()
        for i, b in zip(q[s].tolist(), free[s].tolist()):
            if b >= 0 and i % 2 == s % 2:
                ex.add((min(i, b), max(i, b)))
            for j in (TC - 1, TC, nb + pt - 1, nb + pt):
                if j != i:
                    ex.add((min(i, j), max(i, j)))
            j = next(j for j in range(nt) if j != i and (min(i, j) * nt + max(i, j)) % 32 == 31)
            ex.add((min(i, j), max(i, j)))
        per.append(sorted(ex))
    lists = per if stride == "padded" else [per[0]] * B
    exm = torch.zeros(B, nt, nt, dtype=torch.bool)
    for s in range(B):
        for i, j in lists[s]:
            exm[s, i, j] = exm[s, j, i] = True
    assert any((i * nt + j) % 32 == 31 for i, j in lists[0])
    if stride == "padded":
        words = no_contact_masks(per, B, nt)
        W = words.shape[1]
        nc = torch.full((B, W + 13), -1, dtype=torch.int32)
        nc[:, :W] = words
        body = check_nearest(sc, dtype, md, q, nc=nc.cuda(), stride=W + 13, excluded=exm)
    else:
        body = check_nearest(sc, dtype, md, q, nc=no_contact_masks(per[0], 1, nt).cuda(), stride=0, excluded=exm)
    for s in range(B):
        for i, b in zip(q[s].tolist(), body[s].tolist()):
            assert b < 0 or not bool(exm[s, i, b])
    assert int((body != free).sum()) >= 3
