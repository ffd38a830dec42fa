"""GPU: the contact walk (lcpb200_contacts, csrc/lcp_contacts.cuh) at its chunk, capacity, batch-stride and vertex-count
limits, against the float64 host restatement (tests/contact_ref.py).

Every test calls lcpb200_contacts directly and names the walk it runs: the circle walk (no feat), the polygon walk
(feat) and the mask walk (feat and no_contact), each with the geometry kernel unless stated.
* Enumeration: all-contact scenes (every pair a contact) give exactly the lexicographic pair list at 1023-2049
  pairs (one to three 1024-pair chunks, rows ending inside a thread's 4 items), 2.1 M pairs in 2 049 chunks, one
  circle against 3 000 obstacles (the row clamp), no circles, and one body (no pair: finite padding geometry).
* Mask addressing: random masks over half of all nt * nt bits (bit 31 of many words, bits with i >= j,
  obstacle-obstacle bits), nt not a multiple of 32; a BatchedWorld whose excluded pairs all sit on bit 31.
* Capacity: truncated prefixes, cap = 1, a cap that splits a two-point manifold, the padding, a zero-contact scene
  inside a busy batch.
* Several scenes per CTA: B = 2 (8 SMs) + 5 scenes, B cap beyond the geometry kernel's grid; bitwise equal to the
  same scenes launched at most 8 SMs at a time, sampled scenes against the restatement.
* nv = 256: features naming edges >= 128 and 255, _hull_torch from them, padding by a repeated vertex anywhere.
* Exact rule boundaries and ties in both dtypes; argument checks; one-body worlds.
Tolerances: lists and feat exactly; geometry to 1e-12 x the coordinate scale in float64 and 2e-5 x the coordinate
scale in float32 on scenes whose decisions are exact in float32.
"""
import ctypes

import numpy as np
import pytest
import torch

from tests import contact_ref as cr

pytestmark = pytest.mark.gpu
f64, f32 = torch.float64, torch.float32
DTYPES = [f64, f32]
WALKS = ["circle", "polygon", "mask"]
GEO = ("normal", "p1", "p2", "pen", "mu", "rest")
F32_MARGIN = 1e-5               # x the coordinate scale: a float32 decision closer to its threshold or tie may differ


def coord_scale(sc):
    return max([1.0] + [float(np.abs(sc[k]).max()) for k in ("pos", "pverts", "overts") if sc[k].size])


def pad_pen(dtype):
    """the penetration of unused slots, -1e30 in dtype"""
    return cr.PAD_PEN if dtype == f64 else float(np.float32(cr.PAD_PEN))


def geo_tol(dtype):
    return 1e-12 if dtype == f64 else 2e-5


def launch(batch, dtype, cap, walk, eps=0.1, geometry=True, mask=None, nv=None, B=None, raw=False):
    """lcpb200_contacts on a batch (contact_ref layout) as `walk`; returns its outputs as numpy arrays (raw: the
    return code instead of raising)"""
    from lcp_physics_b200 import _lib
    lib = _lib.load()
    B = batch["pos"].shape[0] if B is None else B
    nb, npoly, no = batch["pos"].shape[1], batch["pverts"].shape[1], batch["overts"].shape[1]
    nt = nb + npoly + no
    nv = batch["overts"].shape[2] if no else batch["pverts"].shape[2] if npoly else 4 if nv is None else nv
    g = {k: torch.from_numpy(np.ascontiguousarray(v)).to("cuda", dtype) for k, v in batch.items()}
    i32 = lambda *s: torch.full(s, -7, dtype=torch.int32, device="cuda")
    b1, b2, counts = i32(max(B, 1), cap), i32(max(B, 1), cap), i32(max(B, 1))
    feat = i32(max(B, 1), cap) if walk != "circle" else None
    new = lambda *s: torch.full((max(B, 1), cap) + s, 7.0, dtype=dtype, device="cuda")
    geo = [new(2), new(2), new(2), new(), new(), new()] if geometry else [None] * 6
    if walk == "mask":
        words = np.zeros((nt * nt + 31) // 32, np.uint32) if mask is None else mask
        mk = torch.from_numpy(words.view(np.int32)).cuda()
    else:
        mk = None
    rc = lib.lcpb200_contacts(
        _lib.dtype_code(dtype), B, nb, npoly, no, nv, cap, eps,
        *[_lib.ptr(g[k]) for k in cr.KEYS], _lib.ptr(b1), _lib.ptr(b2), _lib.ptr(counts), _lib.ptr(feat),
        *[_lib.ptr(t) for t in geo], _lib.ptr(mk), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    if raw:
        return rc
    _lib.check(rc)
    torch.cuda.synchronize()
    out = dict(b1=b1.cpu().numpy(), b2=b2.cpu().numpy(), counts=counts.cpu().numpy())
    if feat is not None:
        out["feat"] = feat.cpu().numpy()
    if geometry:
        out.update({k: t.cpu().double().numpy() for k, t in zip(GEO, geo)})
    return out


def walks_for(npoly):
    return WALKS if npoly == 0 else WALKS[1:]


def check_scene(out, s, ref, cap, nb, nt, dtype, scale, walk, geometry=True):
    """scene s of a launch against the restatement's result ref: lists, feat and the padding exactly, geometry to
    geo_tol(dtype) x scale"""
    t = cr.truncate(ref, cap, nb, nt)
    assert int(out["counts"][s]) == t["count"], (s, int(out["counts"][s]), t["count"])
    assert np.array_equal(out["b1"][s], t["b1"]) and np.array_equal(out["b2"][s], t["b2"]), s
    if walk != "circle":
        assert np.array_equal(out["feat"][s], t["feat"]), s
    if not geometry:
        return
    n = min(ref["count"], cap)
    for k in GEO:
        assert np.abs(out[k][s, :n] - ref[k][:n]).max(initial=0.0) <= geo_tol(dtype) * scale, (s, k)
    assert np.all(out["pen"][s, n:] == pad_pen(dtype))
    for k in GEO:
        assert np.isfinite(out[k][s]).all(), (s, k)


def scattered(sc, gap=300.0):
    """the scene with every body moved apart (same shapes, no contact)"""
    out = dict(sc)
    k = 0
    for key, ck in (("pos", None), ("pverts", "pcen"), ("overts", "oref")):
        n = sc[key].shape[0]
        shift = gap * (np.arange(n) + k + 1)[:, None]
        off = np.concatenate([shift, np.full((n, 1), -gap * (k + 1))], 1)
        out[key] = sc[key] + (off if key == "pos" else off[:, None, :])
        if ck:
            out[ck] = sc[ck] + off
        k += n
    return out


# ---------------------------------------------------------------------------------------------------- enumeration
ENUM_SHAPES = [cr.shape_for_pairs(P) for P in (1023, 1024, 1025, 2047, 2048, 2049)] + [(1, 3000), (2049, 0)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("walk", WALKS)
@pytest.mark.parametrize("shape", ENUM_SHAPES, ids=lambda s: "%dx%d" % s)
def test_all_contact_scenes_give_the_lexicographic_pair_list(shape, walk, dtype):
    nb, no = shape
    I, J = cr.pair_list(nb, 0, no)
    P = I.shape[0]
    sc = cr.all_contact_scene(nb, no)
    cap = P + 5
    out = launch(cr.stack([sc]), dtype, cap, walk)
    assert int(out["counts"][0]) == P
    assert np.array_equal(out["b1"][0, :P], I) and np.array_equal(out["b2"][0, :P], J)
    assert np.all(out["b1"][0, P:] == 0) and np.all(out["b2"][0, P:] == 1) and np.all(out["pen"][0, P:] == pad_pen(dtype))
    if walk != "circle":
        assert np.all(out["feat"][0] == -1)
    # the geometry kernel's grid-stride loop (2.1 M slots): circle-circle geometry against the restatement
    cc = J < nb
    pen, n, p1, p2 = cr.circle_circle(cr.rounded(sc, dtype)["pos"], cr.rounded(sc, dtype)["rad"], I[cc], J[cc])
    tol = geo_tol(dtype) * 20
    for k, want in (("pen", pen), ("normal", n), ("p1", p1), ("p2", p2)):
        assert np.abs(out[k][0, :P][cc] - want).max(initial=0.0) <= tol, k
    assert all(np.isfinite(out[k][0]).all() for k in GEO)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("walk", WALKS)
def test_one_body_and_one_polygon_pair(walk, dtype):
    """nt = 1 (no pair: count 0, the padding pair (0, 0) with finite geometry) and nb = 0, np = 1, no = 1"""
    sc = cr.make_scene([[0.0, 0.0]], 1.0)
    out = launch(cr.stack([sc]), dtype, 3, walk)
    assert int(out["counts"][0]) == 0 and np.all(out["b1"][0] == 0) and np.all(out["b2"][0] == 0)
    assert np.all(out["pen"][0] == pad_pen(dtype))
    for k in GEO:
        assert np.isfinite(out[k][0]).all(), k
    if walk == "circle":
        return
    sc = cr.make_scene(None, None, [cr.box(0, 0, 4, 4)], [cr.box(-10, -4, 10, 0.25)])
    ref = cr.scene_contacts(sc, 0.1)
    assert ref["count"] == 2
    out = launch(cr.stack([sc]), dtype, 4, walk)
    check_scene(out, 0, ref, 4, 0, 2, dtype, 10.0, walk)


# ---------------------------------------------------------------------------------------------------- mask
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape", [(40, 7), (300, 5)])
def test_mask_excludes_exactly_the_set_bits_with_i_below_j(shape, dtype):
    nb, no = shape
    nt = nb + no
    assert nt % 32
    rng = np.random.default_rng(nt)
    words = rng.integers(0, 1 << 32, (nt * nt + 31) // 32, dtype=np.uint64).astype(np.uint32)   # half of all bits
    assert sum(int(w) >> 31 for w in words) > len(words) // 4                                   # bit 31 of many words
    I, J = cr.pair_list(nb, 0, no)
    keep = ~cr.mask_bits(words, I, J, nt)
    # bits with i >= j and obstacle-obstacle bits are set too, and ignored
    lower = [(b, a) for a in range(nt) for b in range(a + 1) if (words[(b * nt + a) >> 5] >> ((b * nt + a) & 31)) & 1]
    assert len(lower) > nt and any(a >= nb and b > a for a, b in [(i, j) for i in range(nb, nt) for j in range(i + 1, nt)
                                                                  if (words[(i * nt + j) >> 5] >> ((i * nt + j) & 31)) & 1])
    sc = cr.all_contact_scene(nb, no)
    cap = int(keep.sum()) + 3
    out = launch(cr.stack([sc, sc]), dtype, cap, "mask", mask=words)
    for s in range(2):
        assert int(out["counts"][s]) == int(keep.sum())
        assert np.array_equal(out["b1"][s, :cap - 3], I[keep]) and np.array_equal(out["b2"][s, :cap - 3], J[keep])
    # the unmasked polygon walk on the same scene: every pair
    out = launch(cr.stack([sc]), dtype, I.shape[0], "polygon")
    assert np.array_equal(out["b1"][0], I) and np.array_equal(out["b2"][0], J)


def test_world_no_contact_pairs_on_bit_31_match_torch():
    """BatchedWorld(no_contact=...) with every excluded pair on bit 31 of its word (negative as int32)"""
    from lcp_physics_b200.world import BatchedWorld
    nb = 40
    rng = np.random.default_rng(1)
    pos = torch.from_numpy(rng.random((2, nb, 2)) * 20.0)
    excl = [(a, b) for a in range(nb) for b in range(a + 1, nb) if (a * nb + b) % 32 == 31]
    assert len(excl) >= 20
    w = BatchedWorld(pos, 2.5, no_contact=excl, contact_capacity=800, strict_no_penetration=False, device="cuda")
    assert int((w.nc_mask < 0).sum()) >= 20
    counts, b1, b2 = w.find_contacts_torch()
    assert torch.equal(w.counts, counts)
    for s in range(2):
        n = int(counts[s])
        assert torch.equal(w.c_b1[s, :n], b1[s, :n]) and torch.equal(w.c_b2[s, :n], b2[s, :n])
        got = set(zip(w.c_b1[s, :n].tolist(), w.c_b2[s, :n].tolist()))
        assert not got & set(excl)
    full = BatchedWorld(pos, 2.5, contact_capacity=800, strict_no_penetration=False, device="cuda")
    assert bool((full.counts > w.counts).all())                                 # the mask excluded contacts


# ---------------------------------------------------------------------------------------------------- capacity
def _capacity_scenes(walk):
    if walk == "circle":
        busy = cr.all_contact_scene(30, 3)
    else:
        busy = cr.aligned_stack(4)
    return busy, scattered(busy)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("walk", WALKS)
def test_capacity_prefix_padding_and_zero_contact_scene(walk, dtype):
    busy, zero = _capacity_scenes(walk)
    nb, npoly, no = busy["pos"].shape[0], busy["pverts"].shape[0], busy["overts"].shape[0]
    nt = nb + npoly + no
    mask = None
    if walk == "mask":                                                          # exclude some contacts
        mask = cr.mask_words(nt, [(2, 3), (8, 10), (0, 5)])
    batch = cr.stack([busy, zero, busy])
    ref = cr.scene_contacts(cr.rounded(busy, dtype), 0.1, mask)
    rz = cr.scene_contacts(cr.rounded(zero, dtype), 0.1, mask)
    assert rz["count"] == 0 and ref["count"] > 10
    caps = [1, ref["count"] // 3, ref["count"], ref["count"] + 9]
    if walk != "circle":                                                        # split a two-point manifold
        pairs = list(zip(ref["b1"].tolist(), ref["b2"].tolist()))
        k = next(k for k in range(len(pairs) - 1) if pairs[k] == pairs[k + 1] and pairs[k][0] >= nb)
        caps.append(k + 1)
    for cap in caps:
        out = launch(batch, dtype, cap, walk, mask=mask)
        for s, r in ((0, ref), (1, rz), (2, ref)):
            check_scene(out, s, r, cap, nb, nt, dtype, 60.0, walk)


# ---------------------------------------------------------------------------------------------------- scenes per CTA
def _cta_batch(B, npoly):
    """B scenes of one shape (20 circles, npoly polygons, 2 obstacles, nv = 6) cycling through: bodies far apart,
    a sparse random scene (few or no contacts), a clump with more contacts than the capacity, a dense random scene"""
    nb, no = 20, 2
    scs = []
    for s in range(B):
        kind = s % 4
        if kind == 0:
            sc = scattered(cr.random_scene(s, nb, npoly, no, 60.0))
        elif kind == 1:
            sc = cr.random_scene(s, nb, npoly, no, 400.0)
        elif kind == 2:
            sc = cr.all_contact_scene(nb, no, nv=6, seed=s)
            pv = np.array([cr.box(-3.0 - k, -3.0, 3.0 + k, 3.0, 6) for k in range(npoly)]).reshape(npoly, 6, 2)
            sc = cr.make_scene(sc["pos"], sc["rad"], pv, sc["overts"], nv=6, seed=s)
        else:
            sc = cr.random_scene(s, nb, npoly, no, 50.0)
        scs.append(sc)
    return cr.stack(scs)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("npoly", [0, 4])
def test_several_scenes_per_cta(npoly, dtype):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    grid = 8 * sms
    B = 2 * grid + 5
    cap = grid * 256 // B + 8
    assert B * cap > grid * 256                                                # the geometry kernel strides too
    batch = _cta_batch(B, npoly)
    nb, no = 20, 2
    nt = nb + npoly + no
    mask = cr.mask_words(nt, [(0, 1), (1, nb), (nb - 1, nb + npoly)])
    sample = sorted({0, grid - 1, grid, 2 * grid, B - 1} | set(range(1, B, 59)))          # 59: every kind of scene
    seen = set()
    for walk in walks_for(npoly):
        mk = mask if walk == "mask" else None
        out = launch(batch, dtype, cap, walk, mask=mk)
        for a in range(0, B, grid):                                            # at most 8 SMs scenes per launch
            part = {k: v[a:a + grid] for k, v in batch.items()}
            sub = launch(part, dtype, cap, walk, mask=mk)
            for k, v in sub.items():
                assert np.array_equal(out[k][a:a + grid], v), (walk, a, k)
        checked = 0
        for s in sample:
            sc = cr.rounded(cr.scene_of(batch, s), dtype)
            ref = cr.scene_contacts(sc, 0.1, mk)
            seen.add("empty" if ref["count"] == 0 else "over" if ref["count"] > cap else "some")
            if dtype == f32 and ref["margin"] <= F32_MARGIN * coord_scale(sc):
                continue                                                       # a float32 decision may differ
            check_scene(out, s, ref, cap, nb, nt, dtype, coord_scale(sc), walk)
            checked += 1
        assert checked >= (len(sample) if dtype == f64 else len(sample) // 3), (walk, checked)
    assert seen == {"empty", "some", "over"}


# ---------------------------------------------------------------------------------------------------- nv = 256
def _as_world(out, batch, dtype, nv):
    from lcp_physics_b200.world import BatchedWorld
    g = lambda k: torch.from_numpy(batch[k]).to("cuda", dtype)
    w = object.__new__(BatchedWorld)
    B, nb, npoly, no = batch["pos"].shape[0], batch["pos"].shape[1], batch["pverts"].shape[1], batch["overts"].shape[1]
    w.nb, w.np, w.no, w.nv = nb, npoly, no, nv
    w.p = torch.cat([torch.zeros(B, nb + npoly, 1, dtype=dtype, device="cuda"), torch.cat([g("pos"), g("pcen")], 1)], 2)
    w.rad, w.fric_coeff, w.restitution = g("rad"), g("fric"), g("rest")
    w.pfric, w.prest, w.ov, w.oref, w.ofric, w.orest = g("pfric"), g("prest"), g("overts"), g("oref"), g("ofric"), g("orest")
    t = lambda k: torch.from_numpy(out[k]).cuda()
    return w._geometry_torch(t("b1"), t("b2"), t("feat"), g("pverts"))


@pytest.mark.parametrize("dtype", DTYPES)
def test_256_gons_name_edges_past_127(dtype):
    sc = cr.gon_scene()
    batch = cr.stack([sc])
    out = launch(batch, dtype, 8, "polygon")
    n = int(out["counts"][0])
    fs = [cr.unpack_feat(int(f)) for f in out["feat"][0, :n]]
    assert 255 in {f["ie"] for f in fs} | {f["re"] for f in fs}
    assert max(f["re"] for f in fs) >= 128 and max(f["ie"] for f in fs) >= 128
    if dtype == f64:                                                           # the restatement: float64 only
        check_scene(out, 0, cr.scene_contacts(sc, 0.1), 8, 0, 4, dtype, 40.0, "polygon")
    got = _as_world(out, batch, dtype, 256)                                    # _hull_torch decodes the same feat
    for k, a in zip(GEO[:4], got[:4]):
        assert np.abs(a[0, :n].cpu().double().numpy() - out[k][0, :n]).max() <= geo_tol(dtype) * 40, k


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("where", ["first", "last", "middle"])
def test_padding_by_a_repeated_vertex_anywhere(where, dtype):
    base = cr.aligned_stack(4)
    ref = launch(cr.stack([base]), dtype, 64, "polygon")
    n = int(ref["counts"][0])
    assert n > 16

    def edge(V, e):
        return np.concatenate([V[e], V[(e + 1) % V.shape[0]]])

    for nv in (6, 64, 256):
        sc = dict(base)
        sc["pverts"] = np.stack([cr.pad_at(v, nv, where) for v in base["pverts"]])
        sc["overts"] = np.stack([cr.pad_at(v, nv, where) for v in base["overts"]])
        out = launch(cr.stack([sc]), dtype, 64, "polygon")
        assert int(out["counts"][0]) == n
        assert np.array_equal(out["b1"], ref["b1"]) and np.array_equal(out["b2"], ref["b2"])
        for k in GEO:
            assert np.abs(out[k][0, :n] - ref[k][0, :n]).max() <= geo_tol(dtype) * 40, (nv, k)
        polys = lambda s, b: s["pverts"][b - 2] if b - 2 < s["pverts"].shape[0] else s["overts"][b - 2 - s["pverts"].shape[0]]
        for c in range(n):
            f0, f1 = int(ref["feat"][0, c]), int(out["feat"][0, c])
            if f0 < 0:
                assert f1 == -1
                continue
            assert f0 & 31 == f1 & 31, (nv, c)                                 # kind, clip1, ref2
            u0, u1 = cr.unpack_feat(f0), cr.unpack_feat(f1)
            i, j = int(ref["b1"][0, c]), int(ref["b2"][0, c])
            br, bi = (j, i) if u0["ref2"] else (i, j)
            assert np.array_equal(edge(polys(base, br), u0["re"]), edge(polys(sc, br), u1["re"])), (nv, c)
            assert np.array_equal(edge(polys(base, bi), u0["ie"]), edge(polys(sc, bi), u1["ie"])), (nv, c)


def test_vertex_count_limits_are_rejected():
    sc = cr.make_scene(None, None, [cr.box(0, 0, 4, 4, 3)[:3]], nv=3)
    ok = cr.stack([sc])
    assert launch(ok, f64, 4, "polygon", raw=True) == 0
    for nv in (2, 257):
        bad = dict(ok)
        V = np.zeros((1, 1, nv, 2))
        bad["pverts"] = V
        assert launch(bad, f64, 4, "polygon", raw=True) != 0, nv
        bad = cr.stack([cr.make_scene([[0.0, 0.0]], 1.0, None, [cr.box(-2, -2, 2, 2)])])
        bad["overts"] = np.zeros((1, 1, nv, 2))
        assert launch(bad, f64, 4, "circle", raw=True) != 0, nv


# ---------------------------------------------------------------------------------------------------- boundaries
@pytest.mark.parametrize("dtype", DTYPES)
def test_exact_rule_boundaries(dtype):
    for name, (sc, want) in cr.boundary_scenes(dtype).items():
        nb, npoly, no = sc["pos"].shape[0], sc["pverts"].shape[0], sc["overts"].shape[0]
        ref = cr.scene_contacts(cr.rounded(sc, dtype), 0.125)
        assert ref["count"] == want, name
        for walk in walks_for(npoly):
            out = launch(cr.stack([sc]), dtype, 3, walk, eps=0.125)
            check_scene(out, 0, ref, 3, nb, nb + npoly + no, dtype, 8.0, walk)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("nv", [4, 6])
def test_axis_aligned_stack_ties(nv, dtype):
    sc = cr.aligned_stack(nv)
    ref = cr.scene_contacts(cr.rounded(sc, dtype), 0.1)
    for walk in ("polygon", "mask"):
        out = launch(cr.stack([sc]), dtype, 64, walk)
        check_scene(out, 0, ref, 64, 2, 2 + sc["pverts"].shape[0] + 2, dtype, 60.0, walk)


# ---------------------------------------------------------------------------------------------------- arguments
def test_argument_checks():
    sc = cr.stack([cr.make_scene([[0.0, 0.0], [1.0, 0.0]], 1.0, [cr.box(0, 0, 4, 4)], [cr.box(-9, -9, 9, -8)])])
    from lcp_physics_b200 import _lib
    lib = _lib.load()
    g = {k: torch.from_numpy(v).cuda() for k, v in sc.items()}
    i32 = lambda *s: torch.full(s, -7, dtype=torch.int32, device="cuda")
    b1, b2, feat, counts = i32(1, 8), i32(1, 8), i32(1, 8), i32(1)
    geo = [torch.zeros(1, 8, 2, dtype=f64, device="cuda") for _ in range(3)] + \
        [torch.zeros(1, 8, dtype=f64, device="cuda") for _ in range(3)]
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call(B=1, cap=8, drop=(), ngeo=6, with_feat=True):
        ins = [None if k in drop else _lib.ptr(g[k]) for k in cr.KEYS]
        gp = [_lib.ptr(t) for t in geo[:ngeo]] + [None] * (6 - ngeo)
        return lib.lcpb200_contacts(_lib.dtype_code(f64), B, 2, 1, 1, 4, cap, 0.1, *ins, _lib.ptr(b1), _lib.ptr(b2),
                                    _lib.ptr(counts), _lib.ptr(feat) if with_feat else None, *gp, None, st)

    assert call() == 0
    assert call(with_feat=False) != 0                                         # polygons without feat
    assert call(drop=("oref",)) != 0                                           # obstacles without oref
    for ngeo in range(1, 6):
        assert call(ngeo=ngeo) != 0, ngeo                                      # 1-5 of the 6 geometry outputs
    assert call(cap=0) != 0
    torch.cuda.synchronize()
    for t in (b1, b2, feat, counts):
        t.fill_(-7)
    before = [t.clone() for t in geo]
    assert call(B=0) == 0                                                      # nothing written
    torch.cuda.synchronize()
    assert all(bool((t == -7).all()) for t in (b1, b2, feat, counts))
    assert all(torch.equal(a, b) for a, b in zip(before, geo))


# ---------------------------------------------------------------------------------------------------- one-body worlds
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("nb", [1, 2])
def test_one_body_world_falls_freely_with_finite_gradients(nb, dtype):
    """one ball, and two balls far apart: no contact ever; the world builds, falls as semi-implicit Euler
    (v += g dt, p += v dt) and d p_y(T) / d v_y(0) = T dt"""
    from lcp_physics_b200.world import BatchedWorld
    B, T, g, dt = 3, 10, 10.0, 1.0 / 30
    pos = torch.tensor([[0.0, 0.0], [1000.0, 0.0]][:nb], dtype=dtype).expand(B, nb, 2).contiguous()
    vel = torch.zeros(B, nb, 3, dtype=dtype)
    vel[:, :, 2] = torch.arange(B, dtype=dtype).unsqueeze(1)
    with torch.no_grad():
        w = BatchedWorld(pos, 1.0, vel=vel, gravity=g, dt=dt, device="cuda")
        assert w.cap >= 1 and int(w.counts.max()) == 0
        for _ in range(T):
            w.step()
            assert bool(torch.isfinite(w.c_normal).all() and torch.isfinite(w.c_p1).all())
    vy, py = vel[:, :, 2].double().clone(), torch.zeros(B, nb, dtype=f64)
    for _ in range(T):
        vy = vy + g * dt
        py = py + vy * dt
    tol = 1e-12 if dtype == f64 else 1e-5
    assert float((w.p[:, :, 2].cpu().double() - py).abs().max()) <= tol * float(py.abs().max())
    assert float((w.p[:, :, 1].cpu().double() - pos[:, :, 0].double()).abs().max()) == 0.0
    v0 = vel.cuda().requires_grad_(True)
    w = BatchedWorld(pos, 1.0, vel=v0, gravity=g, dt=dt, device="cuda")
    for _ in range(T):
        w.step()
    w.p[:, :, 2].sum().backward()
    grad = v0.grad.cpu().double()
    assert bool(torch.isfinite(grad).all())
    assert float((grad[:, :, 2] - T * dt).abs().max()) <= tol * T * dt
    assert float(grad[:, :, :2].abs().max()) <= tol * T * dt
