"""GPU: Jacobians and forward-mode derivatives through LCPFunction (the dense path).

1. One lcpb200_backward_batched call with R cotangents equals R lcpb200_backward calls bitwise -- both kernel
   families, every dual-form residency tier, e in {0, 3}, both adjoints, structure reuse and Rsave on and off, a
   mixed batch, R in {1, 7, n}, a small batch (several chunks per scene) and a batch larger than the grid -- and
   vmap(vjp) equals R .backward() calls bitwise.
2. The JVP matches a dense fp64 solve of the linearised KKT system at the saved iterate.
3. jacfwd agrees with jacrev(exact_adjoint=True) along symmetric directions of Q (and with the default adjoint when
   F = 0), and with central differences on converged solves.
4. One jacfwd call equals R torch.func.jvp calls bitwise; forward_ad duals equal torch.func.jvp bitwise.
5. CPU inputs give the CUDA results; fp32 agrees with fp64.
6. Batched primals, second derivatives and bad C arguments raise.
"""
import pytest
import torch

from tests import dual_plan as dp
from tests.helpers import dual_only
from tests.test_gpu_dual_limits import _check_plan, build_tier

pytestmark = pytest.mark.gpu
f64 = torch.float64
NAMES = "Q p G h A b F".split()


def _bits(t):
    return None if t is None else t.view(torch.int32 if t.dtype == torch.float32 else torch.int64)


def _same(a, b):
    return (a is None and b is None) or torch.equal(_bits(a), _bits(b))


def _handle(dtype, inp):
    from lcp_physics_b200 import _lib
    n, m, e = dp.sizes(inp)
    return _lib.get_handle(dtype, n, m, e, torch.cuda.current_device(), torch.cuda.current_stream().cuda_stream)


def _cuda(inp, dtype):
    return [t.to(dtype).cuda().contiguous() for t in inp]


def _forward_raw(hd, ins, Rsave=None, max_iter=10):
    """lcpb200_forward on device inputs: (zhat, nu, lam, slack, status, resid)."""
    from lcp_physics_b200 import _lib
    Q, p, G, h, A, b, F = ins
    B, m, n = G.shape
    e = A.shape[1] if A.dim() > 1 else 0
    mk = lambda *s, d=Q.dtype: torch.empty(*s, dtype=d, device="cuda")
    zhat, lam, slack, nu = mk(B, n), mk(B, m), mk(B, m), (mk(B, e) if e else None)
    status, iters, resid = mk(B, d=torch.int32), mk(B, d=torch.int32), mk(B)
    _lib.check(_lib.load().lcpb200_forward(hd.raw, B, *[_lib.ptr(t) for t in ins], 1e-12, 3, max_iter,
                                           *[_lib.ptr(t) for t in (zhat, nu, lam, slack, status, iters, resid, Rsave)],
                                           None))
    return zhat, nu, lam, slack, status, resid


def _bwd_raw(hd, ins, state, g, flags, Rsave, batched):
    """Every gradient [R, B, ...]: one lcpb200_backward_batched call, or R lcpb200_backward calls."""
    from lcp_physics_b200 import _lib
    lib = _lib.load()
    Q, p, G, h, A, b, F = ins
    zhat, nu, lam, slack = state
    e = A.shape[1] if A.dim() > 1 else 0
    R = g.shape[0]
    outs = [torch.full((R,) + tuple(t.shape), float("nan"), dtype=t.dtype, device="cuda") if t.numel() else None
            for t in (Q, p, G, h, A, b, F)]
    A_ = A if e else None
    common = [_lib.ptr(t) for t in (Q, G, A_, F, zhat, nu, lam, slack)]
    if batched:
        _lib.check(lib.lcpb200_backward_batched(hd.raw, R, G.shape[0], *common, _lib.ptr(g),
                                                *[_lib.ptr(t) for t in outs], _lib.ptr(Rsave), flags, None))
    else:
        for r in range(R):
            _lib.check(lib.lcpb200_backward(hd.raw, G.shape[0], *common, _lib.ptr(g[r]),
                                            *[_lib.ptr(None if t is None else t[r]) for t in outs], _lib.ptr(Rsave),
                                            flags, None))
    torch.cuda.synchronize()
    return outs


def _check_batched_vjp(dtype, inp, Rs, rsave_ok):
    """Batched against sequential, bitwise, for both adjoints, reuse on / off and (dual form only) Rsave on / off."""
    ins = _cuda(inp, dtype)
    hd = _handle(dtype, inp)
    B, n = ins[1].shape
    m = ins[2].shape[1]
    for use_r in ((False, True) if rsave_ok else (False,)):
        Rsave = torch.empty(B, m, m, dtype=dtype, device="cuda") if use_r else None
        state = _forward_raw(hd, ins, Rsave)[:4]
        for R in Rs:
            g = torch.randn(R, B, n, generator=torch.Generator().manual_seed(R), dtype=f64).to(dtype).cuda()
            for flags in (0, 1, 2, 3):
                if flags & 2:
                    _forward_raw(hd, ins, Rsave)                 # the saved structure is this batch's
                one = _bwd_raw(hd, ins, state, g, flags, Rsave, True)
                seq = _bwd_raw(hd, ins, state, g, flags, Rsave, False)
                for k, (x, y) in enumerate(zip(one, seq)):
                    assert _same(x, y), (NAMES[k], R, flags, use_r)


# ------------------------------------------------------------------ 1. batched VJP = sequential, bitwise
DUAL_TIERS = ["f64_m0_nt128", "f64_m0_G_L2", "f64_split_even", "f64_m2", "f64_m2_nondiag",
              "f32_m0_nt256", "f32_split_even", "f32_m2"]


@pytest.mark.parametrize("e", [0, 3])
@pytest.mark.parametrize("name", DUAL_TIERS)
def test_batched_vjp_dual_tiers_bitwise(name, e):
    dtype, inp = build_tier(name, e, 2)                 # B = 2: several chunks per scene
    n = inp[0].shape[1]
    with dual_only():
        plan, _ = _check_plan(dtype, inp)
        _check_batched_vjp(dtype, inp, (1, 7, n), rsave_ok=True)


@pytest.mark.parametrize("e", [0, 3])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_batched_vjp_condensed_bitwise(dtype, e):
    from lcp_physics_b200.scenes import make_scenes
    inp = make_scenes(3, 8, 12, fd=2, e=e, dtype=f64, seed=21)
    assert "condensed KKT: N=" in _handle(dtype, inp).describe()
    _check_batched_vjp(dtype, inp, (1, 7, inp[0].shape[1]), rsave_ok=False)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_batched_vjp_mixed_batch_bitwise(dtype):
    """Structured scenes and scenes with a dense F (the condensed kernel leaves them to the dual form)."""
    from lcp_physics_b200.scenes import make_scenes
    inp = [t.clone() for t in make_scenes(6, 8, 12, fd=2, e=3, dtype=f64, seed=22)]
    m = inp[6].shape[1]
    W = torch.randn(3, m, m, generator=torch.Generator().manual_seed(1), dtype=f64) * 0.05
    inp[6][::2] += torch.bmm(W, W.transpose(1, 2))
    _check_batched_vjp(dtype, inp, (1, 7), rsave_ok=False)


def test_batched_vjp_more_scenes_than_ctas_bitwise():
    dtype, inp = build_tier("f64_m0_nt128", 3, 2)
    with dual_only():
        _, grid = _check_plan(dtype, inp)
        big = dp.engine_scenes(grid + 5, 8, 8, 2, e=3, seed=308)
        _check_batched_vjp(dtype, big, (1, 3), rsave_ok=True)
    from lcp_physics_b200.scenes import make_scenes
    cgrid = int(_handle(torch.float32, make_scenes(1, 8, 12, fd=2)).describe().split("grid<=")[1].split()[0])
    _check_batched_vjp(torch.float32, make_scenes(cgrid + 5, 8, 12, fd=2, dtype=f64, seed=23), (1, 3), rsave_ok=False)


@pytest.mark.parametrize("exact", [False, True])
@pytest.mark.parametrize("family", ["condensed_f32", "dual_f64"])
def test_vmap_vjp_equals_sequential_backward_bitwise(family, exact):
    from lcp_physics_b200 import LCPFunction
    from lcp_physics_b200.scenes import make_scenes
    dtype = torch.float32 if family == "condensed_f32" else f64
    ins = _cuda(make_scenes(3, 8, 12, fd=2, e=3, dtype=f64, seed=24), dtype)
    fn = LCPFunction(max_iter=8, exact_adjoint=exact)
    B, n = ins[1].shape
    g = torch.randn(7, B, n, generator=torch.Generator().manual_seed(2), dtype=f64).to(dtype).cuda()
    zhat, vjp_fn = torch.func.vjp(fn, *ins)
    batched = torch.vmap(vjp_fn)(g)
    leaves = [t.clone().requires_grad_(True) for t in ins]
    z = fn(*leaves)
    for r in range(g.shape[0]):
        seq = torch.autograd.grad(z, leaves, g[r], retain_graph=True)
        for k in range(7):
            assert _same(batched[k][r], seq[k]), (NAMES[k], r)


# ------------------------------------------------------------------ 2. JVP against the linearised KKT system
def _kkt_jvp(prim, tan, zhat, lam, slack, nu, clamp):
    """Tangent of zhat from K [dx; ds; dz; dy] = -(r_x, 0, r_z, r_y) at the saved iterate, in fp64, with ds
    eliminated and the dz rows / columns scaled by min(1, sqrt(d)) (tests/test_gpu_jvp.py's _dense_jvp)."""
    Q, p, G, h, A, b, F = prim
    tQ, tp, tG, th, tA, tb, tF = tan
    n, m = Q.shape[0], G.shape[0]
    e = A.shape[0] if A.dim() > 1 else 0
    rx = tQ @ zhat + tp + tG.t() @ lam
    rz = tG @ zhat - tF @ lam - th
    d = lam / slack
    if clamp:
        d = d.clamp(1e-10, 1e10)
    N = n + m + e
    K = Q.new_zeros(N, N)
    K[:n, :n] = Q
    K[:n, n:n + m] = G.t()
    K[n:n + m, :n] = G
    K[n:n + m, n:n + m] = -(F + torch.diag(1 / d))
    rhs = [rx, rz]
    if e:
        rx += tA.t() @ nu
        K[n + m:, :n] = A
        K[:n, n + m:] = A.t()
        rhs = [rx, rz, tA @ zhat - tb]
    sc = torch.ones(N, dtype=f64, device=Q.device)
    sc[n:n + m] = d.sqrt().clamp_max(1.0)
    y = torch.linalg.solve(sc[:, None] * K * sc[None, :], -sc * torch.cat(rhs))
    return (sc * y)[:n]


def _tangents(ins, R, seed, e):
    gen = torch.Generator().manual_seed(seed)
    out = []
    for k, t in enumerate(ins):
        if k in (4, 5) and e == 0:
            out.append(None)
            continue
        x = torch.randn((R,) + tuple(t.shape), generator=gen, dtype=f64)
        out.append(x.to(t.dtype).to(t.device))
    return out


@pytest.mark.parametrize("e", [0, 3])
@pytest.mark.parametrize("family", ["condensed_f32", "dual_f64_dense"])
def test_jvp_matches_linearised_kkt(family, e):
    from lcp_physics_b200 import solve_jvp_batched
    from lcp_physics_b200.scenes import make_dense_random, make_scenes
    dtype = torch.float32 if family == "condensed_f32" else f64
    inp = make_dense_random(3, 12, 16, e=e, seed=31) if family == "dual_f64_dense" else \
        make_scenes(3, 8, 12, fd=2, e=e, dtype=f64, seed=31)
    ins = _cuda(inp, dtype)
    hd = _handle(dtype, inp)
    if family == "condensed_f32":
        assert "condensed KKT: N=" in hd.describe()
    zhat, nu, lam, slack, status, resid = _forward_raw(hd, ins)
    tan = _tangents(ins, 1, 7, e)
    A_ = ins[4] if e else None
    dz = solve_jvp_batched(ins[0], ins[2], A_, ins[6], zhat, nu, lam, slack, [None if t is None else t[0] for t in tan])
    worst = 0.0
    for s in range(3):
        prim = [t[s].double() if t.dim() > 1 else t for t in ins]
        tg = [torch.zeros(0, dtype=f64) if t is None else t[0, s].double() for t in tan]
        ref = _kkt_jvp(prim, tg, zhat[s].double(), lam[s].double(), slack[s].double(),
                       nu[s].double() if e else None, clamp=False)
        err = float((dz[s].double() - ref).abs().max()) / max(float(ref.abs().max()), 1e-12)
        worst = max(worst, err)
    print("%s e=%d: JVP against the linearised KKT system, worst %.2e of the scene's scale" % (family, e, worst))
    assert worst <= 3e-5, worst


def _ref_errors(ins, state, tan, dz, scenes):
    """Worst error of dz [B, n] against _kkt_jvp over `scenes`, relative to each scene's scale."""
    zhat, nu, lam, slack = state
    e = ins[4].shape[1] if ins[4].dim() > 1 else 0
    worst = 0.0
    for s in scenes:
        prim = [t[s].double() if t.dim() > 1 else t for t in ins]
        tg = [torch.zeros_like(prim[k]) if t is None else t[s].double() for k, t in enumerate(tan)]
        ref = _kkt_jvp(prim, tg, zhat[s].double(), lam[s].double(), slack[s].double(),
                       nu[s].double() if e else None, clamp=False)
        worst = max(worst, float((dz[s].double() - ref).abs().max()) / max(float(ref.abs().max()), 1e-12))
    return worst


def _jvp_raw(hd, ins, state, tan, batched):
    """dz [R, B, n]: one lcpb200_jvp_batched call with every tangent [R, B, ...], or R single-tangent calls."""
    from lcp_physics_b200 import _lib
    zhat, nu, lam, slack = state
    e = ins[4].shape[1] if ins[4].dim() > 1 else 0
    R = next(t.shape[0] for t in tan if t is not None)
    B, n = zhat.shape
    dz = torch.full((R, B, n), float("nan"), dtype=zhat.dtype, device="cuda")
    base = [_lib.ptr(t) for t in (ins[0], ins[2], ins[4] if e else None, ins[6], zhat, nu, lam, slack)]
    lib = _lib.load()
    if batched:
        _lib.check(lib.lcpb200_jvp_batched(hd.raw, R, B, *base, *[_lib.ptr(t) for t in tan], _lib.ptr(dz), None, 0,
                                           None))
    else:
        for r in range(R):
            _lib.check(lib.lcpb200_jvp_batched(hd.raw, 1, B, *base, *[_lib.ptr(None if t is None else t[r]) for t in tan],
                                               _lib.ptr(dz[r]), None, 0, None))
    torch.cuda.synchronize()
    return dz


def _check_jvp(dtype, inp, R, max_iter=5, ref_scenes=(0, 1)):
    """Batched JVP = single-tangent calls bitwise, and the first tangent against the linearised KKT system at the
    saved iterate (max_iter = 5: an interior iterate, where the derivative is well posed)."""
    ins = _cuda(inp, dtype)
    hd = _handle(dtype, inp)
    state = _forward_raw(hd, ins, max_iter=max_iter)[:4]
    e = dp.sizes(inp)[2]
    tan = _tangents(ins, R, 17, e)
    one = _jvp_raw(hd, ins, state, tan, True)
    seq = _jvp_raw(hd, ins, state, tan, False)
    assert _same(one, seq)
    err = _ref_errors(ins, state, [None if t is None else t[0] for t in tan], one[0], ref_scenes)
    print("JVP against the linearised KKT system: %.2e" % err)
    assert err <= 3e-5, err


@pytest.mark.parametrize("e", [0, 3])
def test_jvp_along_F_only_dual_form(e):
    """Only a tangent of F (tQ ... tb NULL): r_z is -tF lam alone. Raw entry and jacfwd(argnums=6) against jacrev."""
    from lcp_physics_b200 import LCPFunction
    from lcp_physics_b200.scenes import make_dense_random
    inp = make_dense_random(3, 12, 16, e=e, seed=33)
    ins = _cuda(inp, f64)
    hd = _handle(f64, inp)
    state = _forward_raw(hd, ins)[:4]
    tF = _tangents(ins, 3, 8, e)[6]
    tan = [None] * 6 + [tF]
    dz = _jvp_raw(hd, ins, state, tan, True)
    assert _same(dz, _jvp_raw(hd, ins, state, tan, False))
    for r in range(3):
        err = _ref_errors(ins, state, [None] * 6 + [tF[r]], dz[r], range(3))
        assert err <= 3e-5, (r, err)
    fwd = torch.func.jacfwd(lambda F: LCPFunction(max_iter=10)(*ins[:6], F))(ins[6])
    rev = torch.func.jacrev(lambda F: LCPFunction(max_iter=10, exact_adjoint=True)(*ins[:6], F))(ins[6])
    err = float((fwd - rev).abs().max()) / float(rev.abs().max())
    print("F only: jacfwd vs exact jacrev %.2e" % err)
    assert err <= 1e-4, err


@pytest.mark.parametrize("name", ["f64_m0_nt256", "f64_split_even", "f64_m2", "f32_split_even", "f32_m2"])
def test_jvp_dual_tiers(name):
    """Every residency mode of lcp_jvp_kernel: B = 2 (one tangent per chunk) and B = grid (all R per work item)."""
    dtype, inp = build_tier(name, 3, 2)
    with dual_only():
        _, grid = _check_plan(dtype, inp)
        _check_jvp(dtype, inp, 7)
        _check_jvp(dtype, build_tier(name, 3, grid)[1], 7)


@pytest.mark.parametrize("name", ["f64_split_even", "f64_m2", "f32_split_even", "f32_m2"])
def test_batched_vjp_dual_tiers_several_cotangents_per_item(name):
    """B = grid: one chunk per scene, so every work item solves all R cotangents after one factorisation."""
    dtype, inp = build_tier(name, 3, 2)
    with dual_only():
        _, grid = _check_plan(dtype, inp)
        _check_batched_vjp(dtype, build_tier(name, 3, grid)[1], (7,), rsave_ok=True)


def test_jvp_mixed_batch():
    """fp32: structured scenes on the condensed kernel, dense-F scenes handed to the dual form (done / skip)."""
    from lcp_physics_b200.scenes import make_scenes
    inp = [t.clone() for t in make_scenes(6, 8, 12, fd=2, e=3, dtype=f64, seed=22)]
    m = inp[6].shape[1]
    W = torch.randn(3, m, m, generator=torch.Generator().manual_seed(1), dtype=f64) * 0.05
    inp[6][::2] += torch.bmm(W, W.transpose(1, 2))
    assert "condensed KKT: N=" in _handle(torch.float32, inp).describe()
    _check_jvp(torch.float32, inp, 7, ref_scenes=range(6))


@pytest.mark.parametrize("e", [0, 3])
def test_dual_form_contact_jvp_error_is_the_backwards(e):
    """fp64 contact scenes at a converged iterate (d = lam / s spans about 1e+-16): the dual form's JVP and the existing
    exact-adjoint backward (R = n one-hot cotangents, J t assembled from the gradients) are compared with the same
    linearised KKT reference. The JVP is no less accurate than the backward: the error is the dual form's
    conditioning at that iterate, shared by both directions, not the JVP's."""
    from lcp_physics_b200 import solve_backward
    from lcp_physics_b200.scenes import make_scenes
    inp = make_scenes(3, 8, 12, fd=2, e=e, dtype=f64, seed=31)
    ins = _cuda(inp, f64)
    hd = _handle(f64, inp)
    state = _forward_raw(hd, ins)[:4]
    zhat, nu, lam, slack = state
    B, n = zhat.shape
    tan = [None if t is None else t[0] for t in _tangents(ins, 1, 7, e)]
    tan[0] = 0.5 * (tan[0] + tan[0].transpose(1, 2))            # the backward's dQ is symmetrised
    dz = _jvp_raw(hd, ins, state, [None if t is None else t[None] for t in tan], True)[0]
    Jt = torch.zeros(B, n, dtype=f64, device="cuda")
    for i in range(n):
        g = torch.zeros(B, n, dtype=f64, device="cuda")
        g[:, i] = 1
        grads = solve_backward(ins[0], ins[2], ins[4] if e else None, ins[6], zhat, nu, lam, slack, g,
                               exact_adjoint=True)
        for gk, tk in zip(grads, tan):
            if gk is not None and tk is not None:
                Jt[:, i] += (gk * tk).reshape(B, -1).sum(1)
    ej = _ref_errors(ins, state, tan, dz, range(B))
    eb = _ref_errors(ins, state, tan, Jt, range(B))
    print("fp64 contacts e=%d, converged: JVP %.2e, backward %.2e of the scale against the reference" % (e, ej, eb))
    assert ej <= 3 * eb + 3e-5, (ej, eb)


# ------------------------------------------------------------------ 3. jacfwd against jacrev and finite differences
def _sym_fn(fn, e):
    def f(S, p, G, h, A, b, F):
        return fn(0.5 * (S + S.transpose(1, 2)), p, G, h, A if e else torch.tensor([], dtype=S.dtype, device=S.device),
                  b if e else torch.tensor([], dtype=S.dtype, device=S.device), F)
    return f


# fp64 contact scenes at converged iterates: test_dual_form_contact_jvp_error_is_the_backwards
@pytest.mark.parametrize("case", ["dense_e3", "contacts_F0", "dense_e0"])
def test_jacfwd_equals_exact_jacrev(case):
    from lcp_physics_b200 import LCPFunction
    from lcp_physics_b200.scenes import make_dense_random, make_scenes
    inp = make_dense_random(2, 6, 8, e=3 if case == "dense_e3" else 0, seed=41) if case.startswith("dense") else \
        [t.clone() for t in make_scenes(2, 6, 6, fd=2, e=0, dtype=f64, seed=41)]
    if case == "contacts_F0":
        inp[6].zero_()
    e = dp.sizes(inp)[2]
    ins = _cuda(inp, f64)
    if not e:
        ins[4] = torch.zeros(2, 1, ins[0].shape[1], dtype=f64, device="cuda")   # placeholders, not read
        ins[5] = torch.zeros(2, 1, dtype=f64, device="cuda")
    argn = tuple(range(7)) if e else (0, 1, 2, 3, 6)
    fwd = torch.func.jacfwd(_sym_fn(LCPFunction(max_iter=20), e), argnums=argn)(*ins)
    for exact in ((True, False) if case == "contacts_F0" else (True,)):
        rev = torch.func.jacrev(_sym_fn(LCPFunction(max_iter=20, exact_adjoint=exact), e), argnums=argn)(*ins)
        for k, a, b_ in zip(argn, fwd, rev):
            scale = max(float(b_.abs().max()), 1e-12)
            err = float((a - b_).abs().max()) / scale
            print("%s exact=%s %s: jacfwd vs jacrev %.2e" % (case, exact, NAMES[k], err))
            assert err <= 1e-4, (NAMES[k], exact, err)


def test_jvp_matches_central_differences():
    from lcp_physics_b200 import LCPFunction
    from lcp_physics_b200.scenes import make_dense_random
    ins = _cuda(make_dense_random(2, 6, 8, e=3, seed=42), f64)
    fn = LCPFunction(max_iter=40, eps=1e-14)
    fn(*ins)
    keep = (fn.resids < 1e-8)
    assert bool(keep.any()), fn.resids
    tan = [t[0] for t in _tangents(ins, 1, 9, 3)]
    tan[0] = 0.5 * (tan[0] + tan[0].transpose(1, 2))
    _, an = torch.func.jvp(fn, tuple(ins), tuple(tan))
    eps = 1e-6
    fd = (fn(*[x + eps * t for x, t in zip(ins, tan)]) - fn(*[x - eps * t for x, t in zip(ins, tan)])) / (2 * eps)
    scale = float(fd[keep].abs().max())
    err = float((an[keep] - fd[keep]).abs().max()) / scale
    print("JVP against central differences: %.2e of the FD scale" % err)
    assert err < 1e-4, err


# ------------------------------------------------------------------ 4. batched JVP = single calls, bitwise
@pytest.mark.parametrize("e", [0, 3])
@pytest.mark.parametrize("family", ["condensed_f32", "dual_f64"])
def test_batched_jvp_equals_single_jvps_bitwise(family, e):
    from lcp_physics_b200 import LCPFunction
    from lcp_physics_b200.scenes import make_scenes
    dtype = torch.float32 if family == "condensed_f32" else f64
    ins = _cuda(make_scenes(3, 8, 12, fd=2, e=e, dtype=f64, seed=51), dtype)
    if not e:
        ins[4] = ins[5] = torch.tensor([], dtype=dtype, device="cuda")
    fn = LCPFunction(max_iter=8)
    diff = [0, 1, 2, 3, 6] + ([4, 5] if e else [])
    R = 5
    tan = _tangents(ins, R, 11, e)

    def f(*xs):
        full = list(ins)
        for k, x in zip(diff, xs):
            full[k] = x
        return fn(*full)
    prim = tuple(ins[k] for k in diff)
    batched = torch.vmap(lambda *t: torch.func.jvp(f, prim, t)[1])(*[tan[k] for k in diff])
    for r in range(R):
        single = torch.func.jvp(f, prim, tuple(tan[k][r] for k in diff))[1]
        assert _same(batched[r], single), r
    import torch.autograd.forward_ad as fwAD
    with fwAD.dual_level():
        duals = [fwAD.make_dual(ins[k], tan[k][0]) for k in diff]
        dual_out = fwAD.unpack_dual(f(*duals)).tangent
    assert _same(dual_out, torch.func.jvp(f, prim, tuple(tan[k][0] for k in diff))[1])


# ------------------------------------------------------------------ 5. CPU inputs
def test_cpu_inputs_match_cuda():
    from lcp_physics_b200 import LCPFunction
    from lcp_physics_b200.scenes import make_dense_random
    inp = make_dense_random(3, 12, 16, e=0, seed=61)          # a well-posed derivative (see the contact test above)
    res = {}
    for dtype in (torch.float32, f64):
        for dev in ("cpu", "cuda"):
            ins = [t.to(dtype).to(dev) for t in inp]
            fn = LCPFunction(max_iter=10)
            tan = [None if t is None else t[0] for t in _tangents(ins, 1, 12, 0)]
            tan[4] = tan[5] = torch.zeros(0, dtype=dtype, device=dev)
            _, jv = torch.func.jvp(fn, tuple(ins), tuple(tan))
            z, vjp_fn = torch.func.vjp(fn, *ins)
            g = torch.randn(4, *z.shape, generator=torch.Generator().manual_seed(3), dtype=f64).to(dtype).to(dev)
            vj = torch.vmap(vjp_fn)(g)
            assert jv.device.type == dev and all(t.device.type == dev for t in vj)
            res[(dtype, dev)] = [jv.double().cpu()] + [t.double().cpu() for t in vj if t.numel()]   # e == 0: no A, b
    for dtype in (torch.float32, f64):
        for a, b in zip(res[(dtype, "cpu")], res[(dtype, "cuda")]):
            err = float((a - b).abs().max()) / max(float(b.abs().max()), 1e-12)
            assert err <= (1e-4 if dtype == torch.float32 else 1e-10), (dtype, err)
    for a, b in zip(res[(torch.float32, "cuda")], res[(f64, "cuda")]):
        err = float((a - b).abs().max()) / max(float(b.abs().max()), 1e-12)
        print("fp32 against fp64: %.2e" % err)
        assert err <= 1e-3, err


# ------------------------------------------------------------------ 6. errors
def test_batched_primals_and_second_derivatives_raise():
    from lcp_physics_b200 import LCPFunction
    from lcp_physics_b200.scenes import make_scenes
    ins = _cuda(make_scenes(2, 6, 6, fd=2, e=3, dtype=f64, seed=71), f64)
    fn = LCPFunction(max_iter=8)
    with pytest.raises(NotImplementedError):
        torch.vmap(lambda Q: fn(Q, *ins[1:]))(torch.stack([ins[0], ins[0]]))
    tan = tuple(t[0] for t in _tangents(ins, 1, 13, 3))
    with pytest.raises(NotImplementedError):
        torch.func.jvp(lambda *x: torch.func.jvp(fn, x, tan)[1], tuple(ins), tan)
    g = torch.ones(2, ins[1].shape[1], dtype=f64, device="cuda")

    def first(*x):
        return torch.func.vjp(fn, *x)[1](g)[1]
    with pytest.raises(NotImplementedError):
        torch.func.vjp(first, *ins)[1](torch.ones_like(ins[1]))


def test_c_entries_reject_bad_arguments():
    from lcp_physics_b200 import _lib
    from lcp_physics_b200.scenes import make_scenes
    inp = make_scenes(2, 6, 6, fd=2, e=3, dtype=f64, seed=72)
    ins = _cuda(inp, f64)
    hd = _handle(f64, inp)
    lib = _lib.load()
    zhat, nu, lam, slack = _forward_raw(hd, ins)[:4]
    B, n = ins[1].shape
    g = torch.zeros(1, B, n, dtype=f64, device="cuda")
    dz = torch.zeros(1, B, n, dtype=f64, device="cuda")
    base = [_lib.ptr(t) for t in (ins[0], ins[2], ins[4], ins[6], zhat, nu, lam, slack)]

    def err():
        return lib.lcpb200_last_error_string().decode()
    assert lib.lcpb200_backward_batched(hd.raw, 0, B, *base, _lib.ptr(g), *[None] * 7, None, 0, None) != 0
    assert "R >= 1" in err()
    assert lib.lcpb200_backward_batched(hd.raw, 1, B, *base, _lib.ptr(g), *[None] * 7, None, 4, None) != 0
    assert "flags" in err()
    tg = [None] * 7
    assert lib.lcpb200_jvp_batched(hd.raw, 0, B, *base, *tg, _lib.ptr(dz), None, 0, None) != 0
    assert "R >= 1" in err()
    assert lib.lcpb200_jvp_batched(hd.raw, 1, B, *base, *tg, None, None, 0, None) != 0
    assert "dz" in err()
    assert lib.lcpb200_jvp_batched(hd.raw, 1, B, *base, *tg, _lib.ptr(dz), None, 1, None) != 0
    assert "flags" in err()
    assert lib.lcpb200_jvp_batched(hd.raw, 1, B, *base, *tg, _lib.ptr(dz), None, 2, None) == 0
