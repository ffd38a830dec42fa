"""CPU: the banded large-scene kernel's plan and ordering, restated in tests/band_plan.py.

* The plan's widest supported band drops a tier as bodies grow: bwa <= 128 up to 773 bodies, 120 up to 1492,
  112 up to 2173, 104 beyond (an H100's 232448-byte opt-in shared memory).
* Under the window check alone (the admission rule before bwa_max was enforced) four ranges of scenes were
  admitted with a band one tier wider than the plan had sized its band storage, panels and factor blocks for.
  Under the enforced rule every admitted band fits the plan.
* Orderings of pinned scenes, including the ones the GPU tests (tests/test_gpu_band_limits.py) use past each tier.
"""
import numpy as np
import pytest

from tests import band_plan as bp


def _ncap(nb):
    return 3 * nb                                   # a settled pile: about 3 contacts per body


def test_plan_tiers():
    tiers = {}
    for nb in range(2, 2300):
        p = bp.carve_plan(nb, _ncap(nb), 4)
        assert p is not None, nb
        tiers.setdefault(p["bwa_max"], []).append(nb)
    assert {k: (v[0], v[-1]) for k, v in tiers.items()} == {128: (2, 773), 120: (774, 1492), 112: (1493, 2173),
                                                            104: (2174, 2299)}
    # the shared-memory budget: a smaller opt-in limit lowers the tiers, none is above 128 (32 SUBR rows)
    # (100 bodies at a 101376-byte limit: 6800 fixed bytes + 2 x 88 x 64 panel bytes + 97^2 x 8 window bytes fit,
    # the 105^2 window of bwa = 80 does not)
    assert bp.carve_plan(100, 300, 4, optin=101376)["bwa_max"] == 72
    assert all(bp.carve_plan(nb, _ncap(nb), 4, optin=10 ** 7)["bwa_max"] == 128 for nb in (2, 500, 3000))


def test_window_check_alone_admits_bands_past_the_plan():
    """The four windows: (bodies, ordered half bandwidths in bodies, admitted bwa, the plan's bwa_max)."""
    found = {}
    for nb in range(2, 2300):
        p = bp.carve_plan(nb, _ncap(nb), 4)
        bad = tuple(b for b in range(64) if bp.admitted(p, b, old=True) and not bp.admitted(p, b))
        if bad:
            bwa = {bp.band_sizes(b)["bwa"] for b in bad}
            assert len(bwa) == 1
            key = (bad, bwa.pop(), p["bwa_max"])
            found.setdefault(key, []).append(nb)
            for b in bad:
                assert not bp.fits_plan(p, b), (nb, b)
    got = {k: (v[0], v[-1]) for k, v in found.items()}
    assert got == {((43, 44), 136, 128): (2, 58),          # window A (a band of 43 needs >= 44 bodies)
                   ((40, 41, 42), 128, 120): (774, 812),   # B
                   ((37, 38, 39), 120, 112): (1493, 1530),  # C
                   ((35, 36), 112, 104): (2174, 2210)}, got   # D
    # window A also outruns the substitution: 136 band rows, SUBR covers 128
    assert bp.band_sizes(43)["bwa"] > bp.SUBR_ROWS


@pytest.mark.parametrize("optin", [bp.H100_SMEM_OPTIN, 101376, 166912])
def test_every_admitted_band_fits_the_plan(optin):
    for nb in list(range(2, 200)) + list(range(700, 2300, 7)):
        p = bp.carve_plan(nb, _ncap(nb), 4, optin=optin)
        if p is None:
            continue
        for bwb in range(0, 64):
            if bp.admitted(p, bwb):
                assert bp.fits_plan(p, bwb), (optin, nb, bwb)
        # and the widest band the plan sized is admitted (nothing is rejected below it)
        top = max(b for b in range(64) if bp.band_sizes(b)["bwa"] <= p["bwa_max"])
        assert bp.admitted(p, top), (optin, nb, top)


def test_border_rule():
    p = bp.carve_plan(60, 200, 4)
    assert bp.admitted(p, 10, nbd=16) and not bp.admitted(p, 10, nbd=17)
    # degree 12 stays in the band, 13 goes to the border; one-body contacts do not count
    for deg, obst, border in ((12, 0, 0), (13, 0, 1), (12, 5, 0)):
        sc = bp.hubs(1, deg, ring=40, obstacle_per_hub=obst)
        o = bp.order_scene(sc)
        assert o["nbb"] == border and (o["rank"][0] < 0) == bool(border), (deg, obst, o["nbb"])
    # a non-zero entry of A pins its body to the border, whatever its degree
    sc = bp.hubs(1, 3, ring=20)
    A = np.zeros((1, 3 * sc["nb"]))
    A[0, 3 * 5 + 2] = 0.5
    o = bp.order(sc["nb"], sc["body1"], sc["body2"], sc["p1"], sc["p2"], A)
    assert o["nbb"] == 1 and o["rank"][5] == -1 and o["nbd"] == 4


def test_pinned_orderings():
    cases = [  # scene, bodies, bwb, candidate (0 BFS, 1 x, 2 y)
        (bp.lattice(40, 20, bp.FIVE), 800, 40, 1),               # window B
        (bp.lattice(41, 19, bp.SIX), 779, 38, 1),                # bwa 120 = the plan's maximum at 779 bodies
        (bp.hex_pile(40, 38), 1521, 38, 1),                      # window C: config 4's pile, scaled up
        (bp.lattice(122, 18, ((1, 0), (0, 1), (2, 0))), 2196, 36, 1),   # window D
        (bp.lattice(6, 4, bp.FIVE), 24, 7, 2),
    ]
    for sc, nb, bwb, choice in cases:
        o = bp.order_scene(sc)
        assert (sc["nb"], o["bwb"], o["choice"]) == (nb, bwb, choice), (nb, o["bwb"], o["widths"])
        assert sorted(r for r in o["rank"] if r >= 0) == list(range(o["nband"]))
    # a path is ordered end to end by the BFS (two sweeps find an end first)
    pos = np.stack([np.arange(30.0), np.zeros(30)], 1)
    perm = np.random.default_rng(0).permutation(30)
    sc = bp.contacts_from_positions(pos[perm], [(int(np.where(perm == i)[0][0]), int(np.where(perm == i + 1)[0][0]))
                                                for i in range(29)])
    o = bp.order_scene(sc)
    assert o["widths"][0] == 1 and o["bwb"] == 1 and o["choice"] == 0
    # where the three candidates tie, the BFS wins (strictly smaller choice)
    assert bp.order_scene(bp.lattice(4, 1, ((1, 0),)))["choice"] == 0


def test_orderings_of_the_window_scenes():
    # tier windows: the scenes the GPU tests send past the limit
    for sc in (bp.lattice(40, 20, bp.FIVE), bp.hex_pile(40, 38), bp.lattice(122, 18, ((1, 0), (0, 1), (2, 0)))):
        o = bp.order_scene(sc)
        p = bp.carve_plan(sc["nb"], len(sc["body1"]), 1)
        assert bp.admitted(p, o["bwb"], o["nbd"], old=True) and not bp.admitted(p, o["bwb"], o["nbd"])
    # the seeded random graphs at the band limit
    for (nb, seed, md), bwb in bp.WIDE_GRAPHS.items():
        sc = bp.random_graph(nb, seed, mean_deg=md)
        o = bp.order_scene(sc)
        assert (o["bwb"], o["nbd"], o["nband"]) == (bwb, 0, nb), (nb, seed, o["bwb"])
        p = bp.carve_plan(nb, len(sc["body1"]), 4)
        assert bp.admitted(p, bwb) == (bwb <= 42), (nb, seed)
        assert bp.admitted(p, bwb, old=True) == (bwb <= 44), (nb, seed)
    assert bp.band_sizes(40)["bwa"] == 128 and bp.band_sizes(42)["bwa"] == 128 and bp.band_sizes(43)["bwa"] == 136


def test_bfs_structure_sizes():
    # several components, isolated bodies and obstacle-only bodies: all of them are band bodies
    a = bp.lattice(5, 3, bp.FIVE)
    pos = np.concatenate([a["pos"], a["pos"] + 100.0, np.array([[500.0, 0.0], [600.0, 0.0], [700.0, 0.0]])])
    pairs = [(int(i), int(j)) for i, j in zip(a["body1"], a["body2"])]
    pairs += [(i + 15, j + 15) for i, j in pairs]
    sc = bp.contacts_from_positions(pos, pairs, obstacle_pairs=[(31, 0.01), (32, 0.02), (3, 0.01)])
    o = bp.order_scene(sc)
    assert o["nband"] == 33 and o["nbb"] == 0 and o["Nbp"] == 104
    ranks = o["rank"]
    assert sorted(ranks) == list(range(33))
    # components are ordered one after the other
    assert max(ranks[:15]) < min(ranks[15:30]) or max(ranks[15:30]) < min(ranks[:15])
