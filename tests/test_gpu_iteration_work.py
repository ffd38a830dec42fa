"""GPU: the PDIPM forward kernels execute no step whose iterate no output reads.

Every output of the forward (zhat, lam, slack, nu, resid) is the best iterate, and an iterate becomes `best` only in
the iteration that forms its residual. So the last iteration a scene runs ends at its termination tests: it factors
nothing and solves nothing. The factorisations and solves the forward kernels executed are read from the two
counters `Handle.profile()` returns after the phases, summed over the batch. For every scene that enters the loop:

* solves == 2 iters - 1: the initial point, then two (affine + corrector) per step, and iters - 1 steps;
* factorisations == iters on the condensed and banded kernels (one for the initial point, one per step);
* factorisations == iters + 1 on the dual form when a termination test stops the scene before its last iteration:
  that kernel factors K before it runs the tests (pdipm.py:98-102).

A scene without contacts (m == 0, status 2, no iterations) counts one of each; a rejected or singular scene (status
< 0) counts none. Covered: the condensed kernel on the dense API (fp32 / fp64, cfg 3 / cfg 2 shapes, e = 0 / 3, band
and dense LU), the dual form, the engine path with contact-free scenes, a large BatchedWorld pile on the banded
kernel, at max_iter 1, 2 and 10, in batches that mix status 0 with status 1 or 2.
"""
import pytest
import torch

from tests.helpers import dual_only
from tests.test_gpu_cond_band_lu import dense_lu

pytestmark = pytest.mark.gpu
ENGINE_NAMES = ["mass", "inertia", "v", "fext", "normal", "p1", "p2", "mu", "restitution"]
DT = 1.0 / 30
N_DUAL_PHASES = 14            # Handle.profile(): the dual-form phases come first
MAX_ITERS = (1, 2, 10)


def _handle(dtype, n, m, e):
    from lcp_physics_b200 import _lib
    return _lib.get_handle(dtype, n, m, e, torch.cuda.current_device(), torch.cuda.current_stream().cuda_stream)


def _counted(hd, fn):
    """fn() with the handle's counters on: (fn's result, the profile)."""
    hd.profile(True)
    out = fn()
    torch.cuda.synchronize()
    return out, hd.profile(False)


def _expected(status, iters, max_iter, dual=False):
    """(factorisations, solves) the forward must execute for scenes ending with these status and iters."""
    fac = sol = 0
    for st, it in zip(status.tolist(), iters.tolist()):
        if st < 0:
            continue
        if it == 0:                                    # no contacts: the initial solve is the answer
            assert st == 2
            fac, sol = fac + 1, sol + 1
            continue
        assert 1 <= it <= max_iter and (st != 0 or it == max_iter), (st, it)
        fac += it + (1 if dual and st != 0 and it < max_iter else 0)
        sol += 2 * it - 1
    return fac, sol


def _check(prof, status, iters, max_iter, dual=False):
    fac, sol = _expected(status.cpu(), iters.cpu(), max_iter, dual)
    assert (prof["factorisations"], prof["solves"]) == (fac, sol), (max_iter, prof["factorisations"], prof["solves"],
                                                                    fac, sol)


def _mixed(status):
    st = set(status.cpu().tolist())
    return 0 in st and bool(st & {1, 2})


def _dense_counts(nb, nc, fd, e, dtype, dual, B=64):
    from lcp_physics_b200 import solve_forward
    from lcp_physics_b200.scenes import make_scenes
    inp = [t.cuda() for t in make_scenes(B, nb, nc, fd=fd, e=e, dtype=dtype, seed=23)]
    hd = _handle(dtype, 3 * nb, nc * (2 + fd), e)
    for max_iter in MAX_ITERS:
        # eps at the median best residual of a plain run: about half of the scenes stop with status 2, some of them
        # before their last iteration
        base = solve_forward(*inp, max_iter=max_iter)
        eps = float(base[6].double().median())
        for kw in (dict(eps=eps), dict(not_improved_lim=1)):
            out, prof = _counted(hd, lambda: solve_forward(*inp, max_iter=max_iter, **kw))
            assert (sum(list(prof.values())[:N_DUAL_PHASES]) > 0) == dual    # which kernel ran
            if "eps" in kw:
                assert _mixed(out[4]), (max_iter, out[4])
            _check(prof, out[4], out[5], max_iter, dual)


@pytest.mark.parametrize("lu", ["band", "dense"])
@pytest.mark.parametrize("e", [0, 3])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("shape", [(32, 64, 2), (16, 32, 3)], ids=["cfg3", "cfg2"])
def test_condensed_dense_api(shape, dtype, e, lu):
    from lcp_physics_b200 import _lib
    _lib.clear_handles()
    if lu == "dense":
        with dense_lu():
            _dense_counts(*shape, e, dtype, dual=False)
    else:
        _dense_counts(*shape, e, dtype, dual=False)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("e", [0, 3])
def test_dual_form(dtype, e):
    with dual_only():
        _dense_counts(16, 32, 3, e, dtype, dual=True)


def _engine(soa, b1, b2, dtype, mode, max_iter, counts=None):
    from lcp_physics_b200.engines import engine_solve, last_solve_info
    leaves = [soa[k].to(dtype).cuda() for k in ENGINE_NAMES]
    engine_solve(*leaves, b1, b2, DT, mode=mode, max_iter=max_iter, counts=counts)
    info = last_solve_info()
    return info["status"], info["iters"]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("mode", [0, 1])
def test_engine_path(mode, dtype):
    """Contact lists with per-scene counts: whole scenes, partial ones and scenes without contacts."""
    from lcp_physics_b200.scenes import make_contact_soa
    B, nb, nc = 48, 32, 64
    soa = dict(make_contact_soa(B, nb, nc, seed=14))
    fext = torch.zeros(B, 3 * nb, dtype=torch.float64)
    fext[:, 2::3] = 10.0 * soa["mass"]
    soa["fext"] = fext
    b1 = soa["body1"].cuda().unsqueeze(0).expand(B, -1).contiguous()
    b2 = soa["body2"].cuda().unsqueeze(0).expand(B, -1).contiguous()
    counts = torch.tensor([(nc, 0, nc // 2)[k % 3] for k in range(B)], dtype=torch.int32).cuda()
    hd = _handle(dtype, 3 * nb, (4 if mode == 0 else 1) * nc, 0)
    for max_iter in MAX_ITERS:
        for cnt in (None, counts):
            (status, iters), prof = _counted(hd, lambda: _engine(soa, b1, b2, dtype, mode, max_iter, cnt))
            assert (status >= 0).all()
            if cnt is not None:
                assert (iters.cpu()[1::3] == 0).all()
            _check(prof, status, iters, max_iter)


def test_batched_world_banded():
    """bench.py's cfg 4 pile (512 balls on a pinned floor) is solved by the banded kernel, which adds its half
    bandwidth to the `c_gradients` counter."""
    from lcp_physics_b200 import engines as _eng
    from lcp_physics_b200.scenes import make_ball_pile
    from lcp_physics_b200.world import BatchedWorld
    ic = make_ball_pile(2, nballs=512, cols=32, seed=3000, gap=0.05)
    w = BatchedWorld(ic["pos"], ic["rad"], vel=ic["vel"], mass=ic["mass"], restitution=ic["rest"],
                     fric_coeff=ic["fric"], gravity=100.0, static=(0,), dt=DT)
    w.step()
    hd = _handle(torch.float64, w.n, 4 * w.cap, w.ne)
    for max_iter in MAX_ITERS:
        w.max_iter = max_iter
        _, prof = _counted(hd, lambda: w.solve_dynamics(w.dt))
        info = _eng.last_solve_info()
        assert prof["c_gradients"] > 0                 # the banded kernel ran
        assert (info["status"] >= 0).all()
        _check(prof, info["status"], info["iters"], max_iter)
