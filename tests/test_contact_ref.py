"""CPU: the float64 restatement of the contact walk (tests/contact_ref.py) against the CPU oracle
(oracle/polygon_oracle.OracleHullWorld) and itertools, and the scenes tests/test_gpu_contact_limits.py builds pinned
to the properties it relies on (all-contact, chunk and row boundaries, feature edges >= 128, exact rule boundaries)."""
import numpy as np
import pytest
import torch

from tests import contact_ref as cr

f64 = torch.float64


def _oracle_contacts(sc, eps):
    """OracleHullWorld's contact list for a restatement scene: [(normal, p1, p2, pen, i, j)]"""
    from oracle.polygon_oracle import OracleHullWorld
    hv = np.concatenate([sc["pverts"], sc["overts"]])
    cen = np.concatenate([sc["pcen"], sc["oref"]])
    nc, nh = sc["pos"].shape[0], hv.shape[0]
    t = lambda x: torch.as_tensor(x, dtype=f64)
    o = OracleHullWorld(t(sc["pos"]), t(sc["rad"]), torch.zeros(nc, 3), torch.ones(nc), t(sc["rest"]), t(sc["fric"]),
                        [t(v - c) for v, c in zip(hv, cen)], torch.cat([torch.zeros(nh, 1, dtype=f64), t(cen)], 1),
                        torch.zeros(nh, 3), torch.ones(nh), torch.ones(nh),
                        t(np.concatenate([sc["pfric"], sc["ofric"]])), t(np.concatenate([sc["prest"], sc["orest"]])),
                        [False] * nh, n_static=sc["overts"].shape[0], eps=eps)
    return o.contacts


def _from_gpu_polygons(seed, sizes):
    """a scene of tests/test_gpu_polygons.random_scene as a restatement scene"""
    from tests.test_gpu_polygons import random_scene
    nc, npoly, no, spread = sizes
    s = random_scene(seed, nc, npoly, no, spread)
    sc = cr.make_scene(s["pos"].numpy(), s["rad"].numpy(), s["polys"].numpy().reshape(npoly, 6, 2),
                       s["obst"].numpy().reshape(no, 6, 2), nv=6)
    sc["pfric"], sc["ofric"] = s["pfric"].numpy(), s["ofric"].numpy()
    return sc


def _assert_equals_oracle(sc, eps, scale):
    res = cr.scene_contacts(sc, eps)
    orc = _oracle_contacts(sc, eps)
    assert res["count"] == len(orc)
    assert list(zip(res["b1"].tolist(), res["b2"].tolist())) == [(c[4], c[5]) for c in orc]
    for k, c in enumerate(orc):
        for a, b in ((res["normal"][k], c[0]), (res["p1"][k], c[1]), (res["p2"][k], c[2])):
            assert np.abs(a - b.numpy()).max() < 1e-12 * scale, k
        assert abs(res["pen"][k] - float(c[3])) < 1e-12 * scale, k
    nb = sc["pos"].shape[0]
    assert all((f >= 0) == (i >= nb) for f, i in zip(res["feat"].tolist(), res["b1"].tolist()))
    return res


@pytest.mark.parametrize("sizes", [(3, 8, 2, 60.0), (10, 36, 4, 140.0)])
def test_restatement_equals_oracle_on_random_scenes(sizes):
    two = 0
    for seed in range(100, 104):
        res = _assert_equals_oracle(_from_gpu_polygons(seed, sizes), 0.1, sizes[3])
        kinds = [cr.unpack_feat(f)["kind"] for f in res["feat"].tolist() if f >= 0]
        two += sum(1 for k in kinds if k >= 2)
    assert two > 0                                                  # clipped points, not only incident endpoints


@pytest.mark.parametrize("nv", [4, 6])
def test_restatement_equals_oracle_on_aligned_stack(nv):
    """integer coordinates, exact ties in the SAT scans, the support vertices, ref2 and the incident edges"""
    res = _assert_equals_oracle(cr.aligned_stack(nv), 0.1, 40.0)
    feats = [cr.unpack_feat(f) for f in res["feat"].tolist() if f >= 0]
    assert len(feats) >= 16 and any(f["ref2"] for f in feats) and any(not f["ref2"] for f in feats)
    assert res["margin"] == 0.0                                    # ties


def test_gon_scene_equals_oracle_and_names_high_edges():
    sc = cr.gon_scene()
    res = _assert_equals_oracle(sc, 0.1, 40.0)
    feats = [cr.unpack_feat(f) for f in res["feat"].tolist()]
    edges = {f["re"] for f in feats} | {f["ie"] for f in feats}
    assert 255 in edges and max(f["re"] for f in feats) >= 128 and max(f["ie"] for f in feats) >= 128
    assert {f["ref2"] for f in feats} == {0, 1} and {f["kind"] for f in feats} >= {0, 1, 3}


@pytest.mark.parametrize("shape", [(33, 0, 15), (1, 0, 1024), (41, 0, 5), (46, 0, 22), (1, 0, 2048), (1, 0, 2049),
                                   (7, 5, 3), (0, 1, 1), (1, 0, 0), (2, 0, 0), (0, 3, 0), (1, 0, 3000)])
def test_enumeration_equals_itertools(shape):
    I, J = cr.pair_list(*shape)
    assert list(zip(I.tolist(), J.tolist())) == cr.pair_list_itertools(*shape)
    assert I.shape[0] == cr.n_pairs(*shape)


def test_chunk_boundary_shapes():
    for P in (1023, 1024, 1025, 2047, 2048, 2049):
        nb, no = cr.shape_for_pairs(P)
        assert cr.n_pairs(nb, 0, no) == P
    # rows that end inside a thread's 4 items: row starts at every residue mod 4
    for nb, no in (cr.shape_for_pairs(1023), cr.shape_for_pairs(1025), cr.shape_for_pairs(2047)):
        assert {s % 4 for s in cr.row_starts(nb, 0, no)} == {0, 1, 2, 3}
    assert cr.n_pairs(2049, 0, 0) == 2049 * 2048 // 2 and -(-cr.n_pairs(2049, 0, 0) // cr.CHUNK) == 2049


@pytest.mark.parametrize("shape", [(40, 0), (33, 15), (1, 30), (20, 1)])
def test_all_contact_scenes_are_all_contact(shape):
    nb, no = shape
    sc = cr.all_contact_scene(nb, no)
    res = cr.scene_contacts(sc, 0.1)
    I, J = cr.pair_list(nb, 0, no)
    assert np.array_equal(res["b1"], I) and np.array_equal(res["b2"], J)
    assert res["pen"].min() > 1.0                                  # deep: all-contact in float32 too


def test_mask_reads_only_bits_with_i_below_j():
    nb, no = 20, 5
    nt = nb + no
    sc = cr.all_contact_scene(nb, no)
    rng = np.random.default_rng(0)
    pairs = [(a, b) for a in range(nt) for b in range(nt) if rng.random() < 0.5]
    w = cr.mask_words(nt, pairs)
    assert any(int(x) >> 31 for x in w)                           # bit 31 of a word
    res = cr.scene_contacts(sc, 0.1, mask=w)
    ex = {(a, b) for a, b in pairs if a < b}
    want = [(i, j) for i, j in cr.pair_list_itertools(nb, 0, no) if (i, j) not in ex]
    assert list(zip(res["b1"].tolist(), res["b2"].tolist())) == want
    # bits with i >= j and obstacle-obstacle bits alone exclude nothing
    w2 = cr.mask_words(nt, [(b, a) for a, b in cr.pair_list_itertools(nb, 0, no)] + [(a, a) for a in range(nt)]
                       + [(nb, nb + 1), (nb + 2, nb + 4)])
    assert cr.scene_contacts(sc, 0.1, mask=w2)["count"] == cr.n_pairs(nb, 0, no)


def test_truncation_and_padding_follow_the_header():
    sc = cr.all_contact_scene(6, 2)
    res = cr.scene_contacts(sc, 0.1)
    n = res["count"]
    t = cr.truncate(res, 5, 6, 8)
    assert t["count"] == n == 27 and t["b1"].tolist() == res["b1"][:5].tolist() and t["b2"].tolist() == res["b2"][:5].tolist()
    t = cr.truncate(res, n + 7, 6, 8)
    assert t["b1"][n:].tolist() == [0] * 7 and t["b2"][n:].tolist() == [1] * 7
    assert t["feat"][n:].tolist() == [-1] * 7 and t["pen"][n:].tolist() == [cr.PAD_PEN] * 7
    t = cr.truncate(dict(count=0, b1=[], b2=[], feat=[], pen=[]), 3, 0, 2)
    assert t["feat"].tolist() == [0] * 3 and t["b2"].tolist() == [1] * 3                       # no circles: feat 0
    t = cr.truncate(dict(count=0, b1=[], b2=[], feat=[], pen=[]), 3, 1, 1)
    assert t["b1"].tolist() == [0] * 3 and t["b2"].tolist() == [0] * 3                         # one body: (0, 0)


@pytest.mark.parametrize("dtype", [f64, torch.float32])
def test_boundary_scenes_sit_on_their_boundary(dtype):
    f = np.float32 if dtype == torch.float32 else np.float64
    eps = 0.125
    for name, (sc, want) in cr.boundary_scenes(dtype).items():
        for k, v in sc.items():
            if k in ("pos", "rad", "pverts", "overts") and (dtype == torch.float32 or "past" not in name):
                assert np.array_equal(v.astype(np.float32).astype(np.float64), v), (name, k)
        assert cr.scene_contacts(cr.rounded(sc, dtype), eps)["count"] == want, name
    sc = cr.boundary_scenes(dtype)
    pen = lambda s: float(s["rad"][0] + s["rad"][1] - np.linalg.norm(s["pos"][0] - s["pos"][1]))
    assert pen(sc["cc_at"][0]) == -eps and pen(sc["cc_past"][0]) == -eps - float(np.spacing(f(2.125)))
    d = lambda s: -s["pos"][0][0] - s["rad"][0]
    assert d(sc["cp_at"][0]) == eps and d(sc["cp_past"][0]) == eps + float(np.spacing(f(1.125)))
    assert sc["sat_at"][0]["pverts"][1][0][0] - 4.0 == eps
    assert sc["sat_past"][0]["pverts"][1][0][0] - 4.0 == eps + float(np.spacing(f(4.125)))
    res = cr.scene_contacts(sc["clip_at"][0], eps)
    assert sorted(res["pen"].tolist()) == [-eps, -0.0625]          # one point exactly at eps
    res = cr.scene_contacts(sc["clip_past"][0], eps)
    assert res["pen"].tolist() == [-0.0625]


@pytest.mark.parametrize("where", ["first", "last", "middle"])
def test_padding_by_a_repeated_vertex_leaves_the_restatement_unchanged(where):
    base = cr.aligned_stack(4)
    ref = cr.scene_contacts(base, 0.1)
    for nv in (6, 64):
        sc = dict(base)
        sc["pverts"] = np.stack([cr.pad_at(v, nv, where) for v in base["pverts"]])
        sc["overts"] = np.stack([cr.pad_at(v, nv, where) for v in base["overts"]])
        res = cr.scene_contacts(sc, 0.1)
        assert np.array_equal(res["b1"], ref["b1"]) and np.array_equal(res["b2"], ref["b2"])
        for k in ("normal", "p1", "p2", "pen"):
            assert np.abs(res[k] - ref[k]).max() <= 1e-12 * 40, (nv, k)
