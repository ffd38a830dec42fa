"""The torch.func protocol of the solves' derivatives, shared by LCPFunction (lcp.py) and engine_solve (engines.py).

Each solve's autograd Function sends its backward through VjpFn and its forward-mode rule through JvpFn. These two
are what vmap sees: a vmap level adds one leading dimension to the cotangents or tangents, so that all R directions
of a jacrev, a jacfwd or a vmap of a vjp / jvp reach ONE batched kernel call, which factors each scene's KKT matrix
once for all of them. What differs between the solves -- the kernel calls and the error texts -- is a Solve.
"""
import math

import torch


class Solve:
    """The per-solve part of VjpFn and JvpFn.
    vjp(dzhat [..., B, n], meta, saved) -> the gradients, each with dzhat's leading dims in front;
    jvp(tangents, meta, saved) -> the tangent of zhat [..., B, n], with the tangents' leading dims in front;
    the first n_tangents arguments of JvpFn after meta are the tangents (None: zero); second, vmap_vjp and vmap_jvp
    are the error texts of a second derivative and of a vmap over the solve's inputs that reaches the VJP or the JVP.
    A plain object, not a tuple: torch.func passes it to apply's rules as it is, where it would flatten and rebuild a
    tuple at every transform level of every call."""

    def __init__(self, vjp, jvp, n_tangents, second, vmap_vjp, vmap_jvp):
        self.vjp, self.jvp, self.n_tangents = vjp, jvp, n_tangents
        self.second, self.vmap_vjp, self.vmap_jvp = second, vmap_vjp, vmap_jvp


def flatten_directions(ts, shapes, dtype, device):
    """The leading-dimension rule of the derivative calls: every t in ts that is not None is [..., *shape], with the
    same leading dims, the R directions of one call. Returns (leading dims, R, ts as contiguous [R, *shape] tensors
    of dtype on device, None kept)."""
    lead = next((tuple(t.shape[:t.dim() - len(s)]) for t, s in zip(ts, shapes) if t is not None), ())
    R = math.prod(lead)
    return lead, R, [None if t is None else t.to(device, dtype).reshape(R, *s).contiguous() for t, s in zip(ts, shapes)]


class VjpFn(torch.autograd.Function):
    """The vector-Jacobian product of a solve: dl/dzhat and the saved solve in, solve.vjp's gradients out."""

    @staticmethod
    def forward(dzhat, solve, meta, *saved):
        return solve.vjp(dzhat, meta, saved)

    @staticmethod
    def setup_context(ctx, inputs, output):
        ctx.second = inputs[1].second

    @staticmethod
    def backward(ctx, *grads):
        raise NotImplementedError(ctx.second)

    @staticmethod
    def vmap(info, in_dims, dzhat, solve, meta, *saved):
        if any(d is not None for d in in_dims[3:]):
            raise NotImplementedError(solve.vmap_vjp)
        # one more leading cotangent dim; apply (not forward) so that an enclosing vmap level batches it again
        outs = VjpFn.apply(dzhat.movedim(in_dims[0], 0), solve, meta, *saved)
        return outs, tuple(None if t is None else 0 for t in outs)


class JvpFn(torch.autograd.Function):
    """The Jacobian-vector product of a solve: solve.n_tangents tangents and the saved solve in, the tangent of
    zhat out."""

    @staticmethod
    def forward(solve, meta, *args):
        k = solve.n_tangents
        return solve.jvp(args[:k], meta, args[k:])

    @staticmethod
    def setup_context(ctx, inputs, output):
        ctx.second = inputs[0].second

    @staticmethod
    def backward(ctx, *grads):
        raise NotImplementedError(ctx.second)

    @staticmethod
    def jvp(ctx, *tangents):
        raise NotImplementedError(ctx.second)

    @staticmethod
    def vmap(info, in_dims, solve, meta, *args):
        k = solve.n_tangents
        if any(d is not None for d in in_dims[2 + k:]):
            raise NotImplementedError(solve.vmap_jvp)
        # one more leading tangent dim; a tangent this level does not batch is the same for every direction
        ts = [None if t is None else (t.movedim(d, 0) if d is not None else t.expand((info.batch_size,) + t.shape))
              for t, d in zip(args[:k], in_dims[2:2 + k])]
        return JvpFn.apply(solve, meta, *ts, *args[k:]), 0
