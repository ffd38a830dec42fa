"""GPU: the block-band LU of the condensed KKT matrix (DESIGN.md section 3.1) computes what the dense LU computes.

Scenes whose contacts join bodies at most a few indices apart have a K = Q + G^T W G whose non-zero 16 x 16 blocks
lie within two blocks of the diagonal; the condensed kernels factor those with the band LU, every other scene with
the dense LU. The band LU skips only products with exact zeros, so every output must be bitwise the one the dense
LU gives (LCPB200_COND_FLAGS bit 4 forces the dense LU for every scene): forward results and all gradients, both
adjoints, on the dense API, the engine path and BatchedWorld. A scene with a long-range contact and scenes with
equality rows take the dense LU.
"""
import contextlib
import os

import numpy as np
import pytest
import torch

from tests.helpers import rel_err

pytestmark = pytest.mark.gpu
DENSE_LU = 4                 # LCPB200_COND_FLAGS bit (cnd::CFLAG_DENSE_LU)
NB, NC = 32, 64              # bench.py cfg 3: 32 bodies on an 8 x 4 grid, 64 contacts
DT = 1.0 / 30
ENGINE_NAMES = ["mass", "inertia", "v", "fext", "normal", "p1", "p2", "mu", "restitution"]


@contextlib.contextmanager
def dense_lu():
    """Fresh handles planned with the dense LU forced for every scene."""
    from lcp_physics_b200 import _lib
    old = os.environ.get("LCPB200_COND_FLAGS")
    os.environ["LCPB200_COND_FLAGS"] = str(int(old or 3) | DENSE_LU)
    _lib.clear_handles()
    try:
        yield
    finally:
        if old is None:
            os.environ.pop("LCPB200_COND_FLAGS", None)
        else:
            os.environ["LCPB200_COND_FLAGS"] = old
        _lib.clear_handles()


def both(fn):
    """fn() with the default plan (band LU where the structure allows it) and with the dense LU forced."""
    from lcp_physics_b200 import _lib
    _lib.clear_handles()
    got = fn()
    with dense_lu():
        ref = fn()
    return got, ref


def assert_same(got, ref, what=""):
    assert len(got) == len(ref)
    for k, (a, b) in enumerate(zip(got, ref)):
        if a is None or b is None:
            assert a is None and b is None, (what, k)
            continue
        a, b = a.detach().cpu().numpy(), b.detach().cpu().numpy()
        assert a.dtype == b.dtype and a.shape == b.shape, (what, k)
        assert np.array_equal(a, b, equal_nan=a.dtype.kind == "f"), (what, k, np.abs(a - b).max())


def dense_solve(inp, g, reuse=True):
    """Forward, then the backward with both adjoints (reusing the forward's structure, and once scanning it
    again): outputs and the seven gradients of each, in one flat list."""
    from lcp_physics_b200 import solve_backward, solve_forward
    Q, p, G, h, A, b, F = [t.cuda() for t in inp]
    saved = {}
    out = solve_forward(Q, p, G, h, A, b, F, max_iter=10, save=saved)
    zhat, nu, lam, slack = out[:4]
    res = list(out)
    for exact in (False, True):
        res += solve_backward(Q, G, A, F, zhat, nu, lam, slack, g.cuda(), saved=saved if reuse else None,
                              exact_adjoint=exact)
    res += solve_backward(Q, G, A, F, zhat, nu, lam, slack, g.cuda(), exact_adjoint=True)   # structure scanned again
    torch.cuda.synchronize()
    return res


def _gz(B, n, dtype, seed=3):
    return torch.randn(B, n, generator=torch.Generator().manual_seed(seed), dtype=torch.float64).to(dtype)


@pytest.mark.parametrize("nb,nc", [(NB, NC), (20, 40), (40, 80)])       # NS = 6, 4 and 8 blocks of K
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_band_lu_dense_api_bitwise(dtype, nb, nc):
    from lcp_physics_b200.scenes import make_scenes
    B = 96 if nb == NB else 32
    inp = make_scenes(B, nb, nc, fd=2, e=0, dtype=dtype, seed=11)
    g = _gz(B, 3 * nb, dtype)
    got, ref = both(lambda: dense_solve(inp, g))
    assert (got[4] >= 0).all()
    assert_same(got, ref, str(dtype))


def _long_range(inp, k):
    """Scene k with its first contact moved from its second body to body NB - 1: that contact couples the first
    and the last block of K, so the scene has no narrow block band."""
    Q, p, G, h, A, b, F = [t.clone() for t in inp]
    rows = [0, NC, NC + 1]                                     # the contact's normal and two friction rows
    cols = G[k, 0].nonzero().flatten().tolist()
    b2 = cols[-1] // 3
    assert b2 != NB - 1 and cols[0] // 3 == 0
    for r in rows:
        G[k, r, 3 * (NB - 1):] = G[k, r, 3 * b2:3 * b2 + 3]
        G[k, r, 3 * b2:3 * b2 + 3] = 0
    return Q, p, G, h, A, b, F


def test_long_range_contact_takes_the_dense_lu():
    from oracle import pdipm_oracle as po
    from lcp_physics_b200.scenes import make_scenes
    B, k = 8, 3
    inp = make_scenes(B, NB, NC, fd=2, e=0, dtype=torch.float64, seed=12)
    assert (inp[2][:, 0].nonzero()[:, 1] // 3).max() < NB - 1
    mixed = _long_range(inp, k)
    g = _gz(B, 3 * NB, torch.float64)
    got, ref = both(lambda: dense_solve(mixed, g))
    assert_same(got, ref, "mixed batch")
    # the other scenes are bitwise what they are in a batch without the long-range scene
    plain = dense_solve(inp, g)
    keep = [s for s in range(B) if s != k]
    assert_same([None if t is None else t[keep] for t in got], [None if t is None else t[keep] for t in plain], "band scenes")
    # and the long-range scene is solved right
    one = tuple(t[k:k + 1] if t.dim() > 1 else t for t in mixed)
    want = po.lcp_forward(*one, max_iter=10, coupled=False, pivot=False)
    assert int(got[4][k]) >= 0
    assert rel_err(got[0][k:k + 1].cpu(), want.zhat).max() < 1e-6


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_equality_rows_take_the_dense_lu(dtype):
    from lcp_physics_b200.scenes import make_scenes
    B = 32
    inp = make_scenes(B, NB, NC, fd=2, e=3, dtype=dtype, seed=13)
    g = _gz(B, 3 * NB, dtype)
    got, ref = both(lambda: dense_solve(inp, g))
    assert_same(got, ref, str(dtype))


@pytest.mark.parametrize("nb,nc", [(NB, NC), (20, 40), (40, 80)])       # NS = 6, 4 and 8 blocks of K
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("mode", [0, 1])
def test_band_lu_engine_path_bitwise(mode, dtype, nb, nc):
    from lcp_physics_b200.engines import engine_solve
    from lcp_physics_b200.scenes import make_contact_soa
    B = 64 if nb == NB else 24
    soa = dict(make_contact_soa(B, nb, nc, seed=14))
    fext = torch.zeros(B, 3 * nb, dtype=torch.float64)
    fext[:, 2::3] = 10.0 * soa["mass"]
    soa["fext"] = fext
    b1, b2 = soa["body1"].cuda(), soa["body2"].cuda()
    gz = _gz(B, 3 * nb, dtype).cuda()

    def run():
        res = []
        for exact in (False, True):
            leaves = [soa[k].to(dtype).cuda().requires_grad_(True) for k in ENGINE_NAMES]
            z, st = engine_solve(*leaves, b1, b2, DT, mode=mode, max_iter=10, exact_adjoint=exact)
            (z * gz).sum().backward()
            torch.cuda.synchronize()
            res += [z, st] + [t.grad for t in leaves]
        return res

    got, ref = both(run)
    assert (got[1] >= 0).all()
    assert_same(got, ref, "mode %d" % mode)


@pytest.mark.parametrize("static", [(), (0,)])
def test_band_lu_batched_world_bitwise(static):
    """The --config world piles: pinned to the floor (equality rows: dense LU) and free (band LU)."""
    from lcp_physics_b200.scenes import make_ball_pile
    from lcp_physics_b200.world import BatchedWorld
    ic = make_ball_pile(32, nballs=24, cols=6, seed=2000, gap=0.05)

    def run():
        w = BatchedWorld(ic["pos"], ic["rad"], vel=ic["vel"], mass=ic["mass"], restitution=ic["rest"],
                         fric_coeff=ic["fric"], gravity=100.0, static=list(static), dt=DT)
        res = []
        for _ in range(4):
            w.step()
            res += [w.p.clone(), w.v.clone()]
        torch.cuda.synchronize()
        assert float(w.counts.float().mean()) > 20
        return res

    got, ref = both(run)
    assert_same(got, ref, str(static))
