"""CPU: the restatement of the reference `World.step_dt` with static obstacles in the reference's formulation
(oracle/obstacle_oracle.py: every obstacle a pinned body) against trajectories recorded from the unmodified
reference (tests/golden/bworld_obstacles.npz: circles in a bin of pinned `Rect`s); and the host-side argument checks
of `BatchedWorld(obstacles=...)`."""
import os

import numpy as np
import pytest
import torch

from oracle.obstacle_oracle import OracleObstacleWorld
from lcp_physics_b200.world import check_obstacles, polygon_centroid, rect_vertices

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bworld_obstacles.npz")


def oracle_world(z, w, post_stab):
    return OracleObstacleWorld(z["pos"][w], z["rad"][w], z["vel"][w], z["mass"][w], z["rest"][w], z["fric"][w],
                               [torch.from_numpy(v) for v in z["obst_verts"]], obstacle_fric=z["obst_fric"],
                               obstacle_rest=z["obst_rest"], obstacle_rot=z["obst_pos"][:, 0], gravity=100.0,
                               dt=1.0 / 30, post_stab=post_stab)


@pytest.mark.parametrize("post_stab", [False, True])
def test_obstacle_oracle_matches_reference_world(post_stab):
    z = np.load(GOLDEN)
    tag = "ps" if post_stab else "nops"
    for w in range(z["pos"].shape[0]):
        world = oracle_world(z, w, post_stab)
        for k in range(25):                          # as tests/test_world_oracle.py: the first 25 recorded steps
            world.step()
            assert len(world.contacts) == int(z[tag + "_nc"][k, w]), (w, k)
            assert abs(world.t - z[tag + "_t"][k, w]) < 1e-12
            assert np.abs(world.p.numpy() - z[tag + "_p"][k, w]).max() < 1e-8, (w, k)
            assert np.abs(world.v.numpy().reshape(-1, 3) - z[tag + "_v"][k, w]).max() < 1e-7, (w, k)


def test_obstacle_oracle_first_contact_list_matches_reference():
    z = np.load(GOLDEN)
    for w in range(z["pos"].shape[0]):
        world = oracle_world(z, w, False)
        n = int(z["first_n"][w])
        assert len(world.contacts) == n
        for c, (nrm, p1, p2, pen, i, j) in enumerate(world.contacts):
            assert (i, j) == (int(z["first_b1"][w, c]), int(z["first_b2"][w, c]))
            for a, key in ((nrm, "normal"), (p1, "p1"), (p2, "p2")):
                assert np.abs(a.numpy() - z["first_" + key][w, c]).max() < 1e-9, key
            assert abs(float(pen) - z["first_pen"][w, c]) < 1e-9


def test_rect_vertices_mirror_reference_rect():
    z = np.load(GOLDEN)
    for k in range(z["obst_pos"].shape[0]):
        rot, x, y = z["obst_pos"][k]
        v = rect_vertices([x, y], z["obst_dims"][k], rot)
        assert np.abs(v.numpy() - z["obst_verts"][k]).max() < 1e-12
        assert np.abs(polygon_centroid(v).numpy() - [x, y]).max() < 1e-12
    ang = torch.tensor(0.3, dtype=torch.float64, requires_grad=True)
    rect_vertices([0.0, 0.0], [2.0, 1.0], ang).sum().backward()
    assert ang.grad is not None


def test_check_obstacles_rejects_bad_polygons():
    sq = rect_vertices([0.0, 0.0], [2.0, 2.0])
    assert check_obstacles(sq.unsqueeze(0), 3).shape == (3, 1, 4, 2)
    assert check_obstacles(torch.stack([sq, sq.flip(0)]).unsqueeze(0).expand(2, -1, -1, -1), 2).shape == (2, 2, 4, 2)
    with pytest.raises(ValueError, match="shape|need vertices"):
        check_obstacles(sq, 1)                                        # [V, 2]: not a list of polygons
    with pytest.raises(ValueError, match="need vertices"):
        check_obstacles(sq.unsqueeze(0).unsqueeze(0).expand(2, -1, -1, -1), 3)   # batch mismatch
    with pytest.raises(ValueError, match="3 vertices"):
        check_obstacles(sq[:2].unsqueeze(0), 1)
    with pytest.raises(ValueError, match="convex"):
        check_obstacles(torch.tensor([[[0.0, 0.0], [2.0, 0.0], [0.5, 0.5], [0.0, 2.0]]], dtype=torch.float64), 1)
    with pytest.raises(ValueError, match="zero area"):
        check_obstacles(torch.tensor([[[0.0, 0.0], [1.0, 0.0], [2.0, 0.0]]], dtype=torch.float64), 1)
    with pytest.raises(ValueError, match="non-finite"):
        check_obstacles(torch.tensor([[[0.0, 0.0], [1.0, 0.0], [0.0, float("nan")]]], dtype=torch.float64), 1)
    with pytest.raises(ValueError, match="no polygon"):
        check_obstacles(torch.zeros(0, 4, 2), 1)


def test_torch_circle_polygon_skips_repeated_vertices():
    """A triangle padded to 4 vertices by repeating one: the torch contact rule (the differentiable path and
    find_contacts_torch) equals the plain triangle's, outside and inside, with finite gradients."""
    from lcp_physics_b200.world import BatchedWorld
    tri = torch.tensor([[0.0, 0.0], [40.0, 0.0], [20.0, 30.0]], dtype=torch.float64)
    padded = torch.cat([tri, tri[2:]]).requires_grad_(True)
    assert check_obstacles(padded.detach().unsqueeze(0), 1).shape == (1, 1, 4, 2)
    c = torch.tensor([[[20.0, -7.0], [20.0, 10.0], [45.0, 5.0], [20.0, 36.0]]], dtype=torch.float64)
    k = torch.zeros(1, 4, dtype=torch.long)
    out = []
    for v in (tri, padded):
        w = object.__new__(BatchedWorld)                      # the torch mirror needs only the obstacle arrays
        w.ov, w.nv = v.unsqueeze(0).unsqueeze(0), v.shape[0]
        out.append(w._circle_polygon_torch(c, k))
    for x, y in zip(*out):
        assert torch.equal(x, y) if x.dtype == torch.bool else torch.allclose(x, y, rtol=0, atol=1e-12)
    assert out[1][0].tolist() == [[False, True, False, False]]
    sum(t.sum() for t in out[1][1:]).backward()
    assert bool(torch.isfinite(padded.grad).all())
    with pytest.raises(ValueError, match="convex"):          # a concave polygon stays rejected behind a repeated vertex
        check_obstacles(torch.tensor([[[0.0, 0.0], [2.0, 0.0], [0.5, 0.5], [0.5, 0.5], [0.0, 2.0]]],
                                     dtype=torch.float64), 1)
