"""The torch.func protocol of the solves' derivatives (lcp_physics_b200/_derivatives.py), without a GPU.

VjpFn and JvpFn are driven through a tiny differentiable solve written in torch, z = K^-1 p, whose VJP and JVP calls
keep the kernel calls' leading-dimension contract: every vmap level adds one leading dim to the cotangents or tangents
of ONE call. Its derivatives are checked against torch's own derivatives of the same solve, and the errors are checked
with the exact texts of LCPFunction and engine_solve.
"""
import pytest
import torch
import torch.autograd.forward_ad as fwAD

from lcp_physics_b200._derivatives import JvpFn, Solve, VjpFn, flatten_directions
from lcp_physics_b200.engines import _ENGINE, _EngineSolveFn
from lcp_physics_b200.lcp import _LCP, LCPFunction

f64 = torch.float64
B, N = 3, 4


def _vjp(dz, saved, calls):
    """dz [..., B, n] -> (dK, dp), each with dz's leading dims in front, in one call."""
    K, z = saved
    lead, R, (g,) = flatten_directions([dz], [z.shape], K.dtype, K.device)
    calls.append(lead)
    lam = torch.linalg.solve(K.mT, g.unsqueeze(-1)).squeeze(-1)           # [R, B, n]
    dK = -lam.unsqueeze(-1) * z.unsqueeze(-2)
    return dK.reshape(lead + K.shape), lam.reshape(lead + z.shape)


def _jvp(tangents, saved, calls):
    """tangents of (K, p), each [..., *shape] or None -> the tangent of z [..., B, n], in one call."""
    K, z = saved
    lead, R, (tK, tp) = flatten_directions(tangents, [K.shape, z.shape], K.dtype, K.device)
    calls.append(lead)
    rhs = torch.zeros((R,) + z.shape, dtype=z.dtype)
    if tp is not None:
        rhs = rhs + tp
    if tK is not None:
        rhs = rhs - (tK @ z.unsqueeze(-1)).squeeze(-1)
    return torch.linalg.solve(K, rhs.unsqueeze(-1)).squeeze(-1).reshape(lead + z.shape)


class _SolveFn(torch.autograd.Function):
    """z = K^-1 p, differentiated only through the shared pair, as _LCPFn and _EngineSolveFn are."""

    @staticmethod
    def forward(K, p, solve, meta):
        return torch.linalg.solve(K, p.unsqueeze(-1)).squeeze(-1)

    @staticmethod
    def setup_context(ctx, inputs, output):
        K, _, ctx.solve, ctx.meta = inputs
        ctx.save_for_backward(K, output)
        ctx.save_for_forward(K, output)

    @staticmethod
    def backward(ctx, dz):
        return (*VjpFn.apply(dz, ctx.solve, ctx.meta, *ctx.saved_tensors), None, None)

    @staticmethod
    def jvp(ctx, tK, tp, _solve, _meta):
        return JvpFn.apply(ctx.solve, ctx.meta, tK, tp, *ctx.saved_tensors)

    @staticmethod
    def vmap(info, in_dims, *args):
        raise NotImplementedError("vmap over the inputs of the solve")


def _reference(K, p):
    return torch.linalg.solve(K, p.unsqueeze(-1)).squeeze(-1)


def _case(seed=0):
    g = torch.Generator().manual_seed(seed)
    K = torch.randn(B, N, N, dtype=f64, generator=g) + 4 * torch.eye(N, dtype=f64)
    p = torch.randn(B, N, dtype=f64, generator=g)
    return K, p


def _toy(solve):
    """The solve with solve's error texts, and the list of the leading dims each VJP / JVP call received (the
    calls are closures: torch.func rebuilds containers passed to apply, but passes callables as they are)."""
    calls = []
    spec = Solve(lambda dz, meta, saved: _vjp(dz, saved, calls), lambda ts, meta, saved: _jvp(ts, saved, calls), 2,
                 solve.second, solve.vmap_vjp, solve.vmap_jvp)
    return (lambda K, p: _SolveFn.apply(K, p, spec, None)), calls


def test_jacrev_and_jacfwd_match_torch():
    K, p = _case()
    f, calls = _toy(_LCP)
    want = torch.func.jacrev(_reference, argnums=(0, 1))(K, p)
    rev = torch.func.jacrev(f, argnums=(0, 1))(K, p)
    assert calls == [(B * N,)]                            # one call for every row of the Jacobian
    fwd = torch.func.jacfwd(f, argnums=(0, 1))(K, p)
    assert calls[1:] == [(B * N * N + B * N,)]            # one call for every column
    for got in (rev, fwd):
        for a, b in zip(got, want):
            assert torch.allclose(a, b, rtol=1e-10, atol=1e-12)


def test_nested_vmap_of_a_vjp_is_one_call():
    K, p = _case(1)
    f, calls = _toy(_ENGINE)
    z, vjp_fn = torch.func.vjp(f, K, p)
    _, want_fn = torch.func.vjp(_reference, K, p)
    g = torch.randn(2, 5, B, N, dtype=f64, generator=torch.Generator().manual_seed(2))
    got = torch.func.vmap(torch.func.vmap(vjp_fn))(g)
    assert torch.allclose(z, _reference(K, p))
    assert calls == [(2, 5)]
    for i in range(2):
        for j in range(5):
            for a, b in zip(got, want_fn(g[i, j])):
                assert torch.allclose(a[i, j], b, rtol=1e-10, atol=1e-12)


def test_vmap_of_a_jvp_expands_the_unbatched_tangent():
    K, p = _case(3)
    f, calls = _toy(_LCP)
    gen = torch.Generator().manual_seed(4)
    tKs = torch.randn(6, B, N, N, dtype=f64, generator=gen)                  # batched by the vmap
    tp = torch.randn(B, N, dtype=f64, generator=gen)                         # the same for every direction
    got = torch.func.vmap(lambda tK: torch.func.jvp(f, (K, p), (tK, tp))[1])(tKs)
    assert calls == [(6,)]
    for r in range(6):
        want = torch.func.jvp(_reference, (K, p), (tKs[r], tp))[1]
        assert torch.allclose(got[r], want, rtol=1e-10, atol=1e-12)


def test_forward_ad_dual_tensors():
    K, p = _case(5)
    f, calls = _toy(_ENGINE)
    gen = torch.Generator().manual_seed(6)
    tK, tp = torch.randn(B, N, N, dtype=f64, generator=gen), torch.randn(B, N, dtype=f64, generator=gen)
    with fwAD.dual_level():
        z = f(fwAD.make_dual(K, tK), fwAD.make_dual(p, tp))
        got = fwAD.unpack_dual(z).tangent
        z_p = f(K, fwAD.make_dual(p, tp))                                     # K carries no tangent: None reaches _jvp
        got_p = fwAD.unpack_dual(z_p).tangent
    assert calls == [(), ()]
    assert torch.allclose(got, torch.func.jvp(_reference, (K, p), (tK, tp))[1], rtol=1e-10, atol=1e-12)
    assert torch.allclose(got_p, torch.func.jvp(lambda q: _reference(K, q), (p,), (tp,))[1], rtol=1e-10, atol=1e-12)


TEXTS = {
    "lcp": (_LCP, "LCPFunction: second derivatives are not implemented",
            "LCPFunction: vmap over the inputs of the solve is not supported; batch scenes along dim 0 instead (vmap "
            "of its vector-Jacobian and Jacobian-vector products -- jacrev, jacfwd -- is supported)",
            "LCPFunction: vmap over the inputs of the solve is not supported; batch scenes along dim 0 instead (vmap "
            "of its vector-Jacobian and Jacobian-vector products -- jacrev, jacfwd -- is supported)"),
    "engine": (_ENGINE, "engine_solve: second derivatives are not implemented",
               "engine_solve: vmap over the inputs of the solve is not supported; batch scenes along dim 0 instead "
               "(vmap of the vector-Jacobian product -- torch.func.vjp, jacrev -- is supported)",
               "engine_solve: vmap over the inputs of the solve is not supported; batch scenes along dim 0 instead "
               "(vmap of the Jacobian-vector product -- torch.func.jvp, jacfwd -- is supported)"),
}


def _raises(fn, text):
    with pytest.raises(NotImplementedError) as e:
        fn()
    assert str(e.value) == text


@pytest.mark.parametrize("name", sorted(TEXTS))
def test_errors_carry_each_solves_text(name):
    solve, second, vmap_vjp, vmap_jvp = TEXTS[name]
    K, p = _case(7)
    f, _ = _toy(solve)
    ones = torch.ones(B, N, dtype=f64)
    # second derivatives: forward over forward, reverse over forward, reverse over reverse
    jvp_p = lambda q: torch.func.jvp(lambda x: f(K, x), (q,), (ones,))[1]
    _raises(lambda: torch.func.jvp(jvp_p, (p,), (ones,)), second)
    _raises(lambda: torch.func.vjp(jvp_p, p)[1](ones), second)
    _raises(lambda: torch.func.vjp(lambda q: torch.func.vjp(lambda x: f(K, x), q)[1](ones)[0], p)[1](ones), second)
    # a saved tensor batched by a vmap level: a vmap over the inputs of the solve
    z = _reference(K, p)
    Ks = K.unsqueeze(0).expand(2, -1, -1, -1)
    _raises(lambda: torch.func.vmap(lambda k: VjpFn.apply(ones, solve, None, k, z))(Ks), vmap_vjp)
    _raises(lambda: torch.func.vmap(lambda k: JvpFn.apply(solve, None, *[None] * solve.n_tangents, k, z))(Ks),
            vmap_jvp)


def test_vmap_over_the_inputs_of_either_solve_raises_before_any_kernel():
    K, p = _case(8)
    lcp_in = (K, p, torch.zeros(B, 2, N, dtype=f64), torch.ones(B, 2, dtype=f64), torch.tensor([], dtype=f64),
              torch.tensor([], dtype=f64), torch.zeros(B, 2, 2, dtype=f64))
    _raises(lambda: torch.func.vmap(lambda q: LCPFunction()(q, *lcp_in[1:]))(K.unsqueeze(0).expand(2, -1, -1, -1)),
            TEXTS["lcp"][2])
    mass = torch.ones(B, 2, dtype=f64)                                       # two bodies, one contact
    body = torch.zeros(1, dtype=torch.int32)
    vec, pt, per_contact = torch.zeros(B, 6, dtype=f64), torch.zeros(B, 1, 2, dtype=f64), torch.zeros(B, 1, dtype=f64)
    rest = (mass, vec, vec, pt, pt, pt, per_contact, per_contact, None, None, body, body + 1, 0.01, 0, 10, False)
    _raises(lambda: torch.func.vmap(lambda m: _EngineSolveFn.apply(m, *rest))(mass.unsqueeze(0).expand(2, -1, -1)),
            "engine_solve: vmap over the inputs of the solve is not supported; batch scenes along dim 0 instead")
