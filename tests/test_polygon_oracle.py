"""CPU: the restatement of the reference `World.step_dt` with dynamic `Rect` / `Hull` bodies and the hull-hull contact
rule (oracle/polygon_oracle.py) against trajectories recorded from the unmodified reference
(tests/golden/bworld_polygons.npz: a Rect sliding down a pinned ramp; a mixed stack of Rects, a pentagon Hull and
circles in a pinned bin), the tie-free recorded scenes, and the host-side polygon helpers of BatchedWorld."""
import os

import numpy as np
import pytest
import torch

from oracle.polygon_oracle import OracleHullWorld
from lcp_physics_b200.world import check_polygons, polygon_centroid, polygon_inertia, rect_vertices

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bworld_polygons.npz")
SCENES = ("slide", "stack")


def oracle_world(z, scene, w, post_stab):
    g = lambda k: z["%s_%s" % (scene, k)][w]
    nv = g("hull_nv")
    verts = [torch.from_numpy(v[:n]) for v, n in zip(g("hull_verts"), nv)]
    return OracleHullWorld(g("pos"), g("rad"), g("vel"), g("mass"), g("rest"), g("fric"), verts, g("hull_p"),
                           g("hull_vel"), g("hull_mass"), g("hull_inertia"), g("hull_fric"), g("hull_rest"),
                           g("hull_is_rect"), n_static=int(z[scene + "_nstatic"]), gravity=100.0, dt=1.0 / 30,
                           post_stab=post_stab)


@pytest.mark.parametrize("scene", SCENES)
def test_polygon_oracle_first_contact_list_matches_reference(scene):
    z = np.load(GOLDEN)
    for w in range(z[scene + "_pos"].shape[0]):
        world = oracle_world(z, scene, w, False)
        n = int(z[scene + "_first_n"][w])
        assert len(world.contacts) == n, (w, len(world.contacts), n)
        for c, (nrm, p1, p2, pen, i, j) in enumerate(world.contacts):
            assert (i, j) == (int(z[scene + "_first_b1"][w, c]), int(z[scene + "_first_b2"][w, c]))
            for a, key in ((nrm, "normal"), (p1, "p1"), (p2, "p2")):
                assert np.abs(a.numpy() - z["%s_first_%s" % (scene, key)][w, c]).max() < 1e-12, (key, w, c)
            assert abs(float(pen) - z[scene + "_first_pen"][w, c]) < 1e-12


@pytest.mark.parametrize("post_stab", [False, True])
@pytest.mark.parametrize("scene", SCENES)
def test_polygon_oracle_matches_reference_world(scene, post_stab):
    z = np.load(GOLDEN)
    tag = "%s_%s_" % (scene, "ps" if post_stab else "nops")
    for w in range(z[scene + "_pos"].shape[0]):
        world = oracle_world(z, scene, w, post_stab)
        for k in range(z[tag + "nc"].shape[0]):
            world.step()
            assert len(world.contacts) == int(z[tag + "nc"][k, w]), (w, k)
            assert abs(world.t - z[tag + "t"][k, w]) < 1e-12
            # the LCP solves agree to ~1e-11 (different linear algebra), as in tests/test_obstacle_oracle.py
            assert np.abs(world.p.numpy() - z[tag + "p"][k, w]).max() < 1e-9, (w, k)
            assert np.abs(world.v.numpy().reshape(-1, 3) - z[tag + "v"][k, w]).max() < 1e-8, (w, k)
        # no recorded hull-hull contact sits on a tie the reference's SAT scan order would settle: the winning edge
        # separation is unique, and so is the choice of the reference body
        assert world.margins and min(min(m) for m in world.margins) > 1e-9, (w, min(min(m) for m in world.margins))


def test_polygon_inertia_and_centroid_mirror_reference_hulls():
    z = np.load(GOLDEN)
    for scene in SCENES:
        for w in range(z[scene + "_pos"].shape[0]):
            for v, n, p, m, inert in zip(*[z["%s_%s" % (scene, k)][w] for k in
                                           ("hull_verts", "hull_nv", "hull_p", "hull_mass", "hull_inertia")]):
                world_v = torch.from_numpy(v) + torch.from_numpy(p[1:])            # padded by a repeated vertex
                cen = polygon_centroid(world_v)
                assert np.abs(cen.numpy() - p[1:]).max() < 1e-9
                got = float(polygon_inertia(world_v - cen, torch.tensor(m, dtype=torch.float64)))
                assert abs(got - inert) < 1e-11 * inert, (got, inert)


def test_check_polygons_orientation():
    sq = rect_vertices([0.0, 0.0], [2.0, 1.0], 0.3)
    assert check_polygons(sq.unsqueeze(0), 2).shape == (2, 1, 4, 2)
    with pytest.raises(ValueError, match="orientation"):
        check_polygons(sq.flip(0).unsqueeze(0), 1)
    with pytest.raises(ValueError, match="polygons: every polygon must be convex"):
        check_polygons(torch.tensor([[[0.0, 0.0], [2.0, 0.0], [0.5, 0.5], [0.0, 2.0]]], dtype=torch.float64), 1)
