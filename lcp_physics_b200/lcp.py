"""Drop-in for `lcp_physics.lcp.lcp.LCPFunction` (reference lcp/lcp.py:8-64).

Same constructor keywords, same call signature `(Q, p, G, h, A, b, F) -> zhat`,
differentiable w.r.t. all seven inputs, same conventions:
  * an empty equality set is passed as 1-D empty tensors for A and b
    (engines.py:59-60, detected like lcp.py:24);
  * a singular Q raises the reference's RuntimeError text (pdipm.py:361-368);
  * an inaccurate result (best residual > 1) PRINTS a warning iff verbose >= 0
    and never raises (pdipm.py:134-135,176-178);
  * inputs are never mutated; dtype and device follow the inputs.

The work is done by hand-written sm_90a kernels behind the C ABI in
include/lcpb200.h. CUDA tensors are solved in place on the current stream; CPU
tensors (what the reference's `World` produces) go through the host-buffer entry
points, which copy in, solve and copy back. There is no CPU fallback.
"""
import torch

from . import _lib
from ._derivatives import JvpFn, Solve, VjpFn, flatten_directions

SINGULAR_Q_MSG = """
lcp Error: Cannot perform LU factorization on Q.
Please make sure that your Q matrix is PSD and has
a non-zero diagonal.
"""

INACCURATE_MSG = """
--------
lcp warning: Returning an inaccurate and potentially incorrect solution.
Some residual is large; the problem may be infeasible or difficult.
Try verbose output and more iterations (max_iter).
--------
"""


def _sizes(Q, p, G, h, A, b, F):
    if G.dim() != 3:
        raise ValueError("G must be [B, nineq, nz]")
    B, m, n = G.shape
    e = A.shape[1] if A.dim() > 1 else 0            # lcp.py:24
    if not (e > 0 or m > 0):
        raise AssertionError("need neq > 0 or nineq > 0")   # lcp.py:25
    if m == 0:
        # lcp.py:25 lets neq > 0, nineq == 0 through, but the reference's pdipm then fails (IndexError in
        # its first get_step): there is no behaviour to mirror
        raise ValueError("lcp_physics_b200 needs at least one inequality row (the reference crashes on nineq == 0)")
    exp = {"Q": (B, n, n), "p": (B, n), "h": (B, m), "F": (B, m, m)}
    for name, t in (("Q", Q), ("p", p), ("h", h), ("F", F)):
        if tuple(t.shape) != exp[name]:
            raise ValueError("%s has shape %s, expected %s" % (name, tuple(t.shape), exp[name]))
    if e > 0 and (tuple(A.shape) != (B, e, n) or tuple(b.shape) != (B, e)):
        raise ValueError("A/b have shapes %s/%s, expected %s/%s"
                         % (tuple(A.shape), tuple(b.shape), (B, e, n), (B, e)))
    return B, n, m, e


def solve_forward(Q, p, G, h, A, b, F, eps=1e-12, not_improved_lim=3, max_iter=10, out=None, save=None):
    """Raw forward: returns (zhat, nus, lams, slacks, status, iters, resid).
    All inputs on one device (CUDA or CPU), same dtype. `out` may hold preallocated
    result tensors (same order; pinned host tensors make the host path's D2H fast).
    `save`: a dict that receives what the backward can reuse -- for CPU inputs a token
    of the state the library retained on the device ("token")."""
    _lib.require_cuda()
    lib = _lib.load()
    B, n, m, e = _sizes(Q, p, G, h, A, b, F)
    dtype, dev = Q.dtype, Q.device
    ins = [t.contiguous() for t in (Q, p, G, h)] + \
          [A.contiguous() if e > 0 else None, b.contiguous() if e > 0 else None, F.contiguous()]
    for t in ins:
        if t is not None and (t.dtype != dtype or t.device != dev):
            raise ValueError("all LCP inputs must share dtype and device")
    on_host = dev.type != "cuda"
    dev_index = torch.cuda.current_device() if on_host else dev.index
    hd = _lib.get_handle(dtype, n, m, e, dev_index,
                         "host" if on_host else torch.cuda.current_stream(dev).cuda_stream)
    if out is not None:
        zhat, nu, lam, slack, status, iters, resid = out
    else:
        mk = lambda *shape, dt=dtype: torch.empty(*shape, dtype=dt, device=dev)
        zhat, lam, slack = mk(B, n), mk(B, m), mk(B, m)
        nu = mk(B, e) if e > 0 else None
        status = mk(B, dt=torch.int32)
        iters = mk(B, dt=torch.int32)
        resid = mk(B)
    if B == 0:
        return zhat, nu, lam, slack, status, iters, resid
    args = [hd.raw, B] + [_lib.ptr(t) for t in ins] + [float(eps), int(not_improved_lim), int(max_iter)] + \
           [_lib.ptr(t) for t in (zhat, nu, lam, slack, status, iters, resid)]
    if on_host:
        hd.host_generation += 1
        _lib.check(lib.lcpb200_forward_host(*args))
        if save is not None:
            save["token"] = (hd, hd.host_generation, B)
    else:
        hd.fwd_generation += 1
        with torch.cuda.device(dev):
            _lib.check(lib.lcpb200_forward(*args, None, _lib.stream_ptr(dev)))
        if save is not None:
            # the library keeps the block structure it found for these inputs; a backward for the SAME inputs
            # may reuse it as long as no other forward ran on this handle in between (LCPB200_BWD_REUSE_STRUCTURE)
            save["struct"] = (hd, hd.fwd_generation, B)
    return zhat, nu, lam, slack, status, iters, resid


def solve_backward(Q, G, A, F, zhat, nu, lam, slack, dl_dzhat, need=(True,) * 7, out=None, saved=None,
                   exact_adjoint=False):
    """Raw backward (lcp.py:37-64): returns (dQ, dp, dG, dh, dA, db, dF); entries
    not needed (or dA/db when e == 0) are None. `out`: preallocated results.
    `saved`: the dict filled by solve_forward(save=...) for the same inputs (host path: the state retained on
    the device; CUDA path: a token that lets the backward reuse the block structure the forward found).
    `exact_adjoint`: False = the reference's behaviour (it re-uses the UN-transposed KKT
    factorisation, which is the true adjoint only when F == 0 -- SURVEY.md F6); True = the
    transposed system (F^T in place of F inside the KKT solve), the exact gradient.
    CUDA inputs take solve_backward_batched with one cotangent; CPU inputs the host-buffer path."""
    if G.device.type == "cuda":
        return solve_backward_batched(Q, G, A, F, zhat, nu, lam, slack, dl_dzhat, need, saved=saved,
                                      exact_adjoint=exact_adjoint, out=out)
    _lib.require_cuda()
    lib = _lib.load()
    B, m, n = G.shape
    e = A.shape[1] if (A is not None and A.dim() > 1) else 0
    dtype = G.dtype
    hd = _lib.get_handle(dtype, n, m, e, torch.cuda.current_device(), "host")
    shapes = [(B, n, n), (B, n), (B, m, n), (B, m), (B, e, n), (B, e), (B, m, m)]
    outs = []
    for k, shp in enumerate(shapes):
        want = need[k] and not (k in (4, 5) and e == 0)
        if out is not None:
            outs.append(out[k] if want else None)
        else:
            outs.append(torch.empty(*shp, dtype=dtype, device=G.device) if want else None)
    if B == 0:
        return tuple(outs)
    ins = [Q.contiguous(), G.contiguous(), A.contiguous() if e > 0 else None, F.contiguous(),
           zhat.contiguous(), nu.contiguous() if e > 0 else None, lam.contiguous(), slack.contiguous(),
           dl_dzhat.contiguous().to(dtype)]
    if _reuses(saved, "token", hd, hd.host_generation, B):
        in_ptrs = [None] * 8 + [_lib.ptr(ins[8])]          # reuse what forward_host left on the device
    else:
        in_ptrs = [_lib.ptr(t) for t in ins]
    hd.host_generation += 1
    _lib.check(lib.lcpb200_backward_host(hd.raw, B, *in_ptrs, *[_lib.ptr(t) for t in outs], 1 if exact_adjoint else 0))
    return tuple(outs)


def _reuses(saved, kind, hd, generation, B):
    """True when `saved`, filled by solve_forward(save=...), holds the token of the last forward on handle hd
    (generation) for B scenes: "struct" for the block structure of the device path, "token" for the state the host
    path retained."""
    return bool(saved) and saved.get(kind) == (hd, generation, B)


def _saved_on(run, home, e, Q, G, A, F, zhat, nu, lam, slack):
    """The saved solve as the batched dense entries take it: contiguous, on the device the call runs on."""
    return [None if t is None else (t.contiguous() if home == run else t.to(run).contiguous())
            for t in (Q, G, A if e > 0 else None, F, zhat, nu if e > 0 else None, lam, slack)]


def _device_call(dev):
    """(device to run on, device the results go back to): CPU inputs run on the current CUDA device."""
    if dev.type == "cuda":
        return dev, dev
    return torch.device("cuda", torch.cuda.current_device()), dev


def solve_backward_batched(Q, G, A, F, zhat, nu, lam, slack, dl_dzhat, need=(True,) * 7, saved=None,
                           exact_adjoint=False, out=None):
    """lcpb200_backward_batched: dl_dzhat [..., B, n] -> (dQ, dp, dG, dh, dA, db, dF), each with dl_dzhat's leading
    dims in front; entries not needed (or dA/db when e == 0) are None. The leading dims are the R cotangents of one
    call: each scene's KKT matrix is factored once for all of them. Slot r equals solve_backward(dl_dzhat[r]).
    CPU inputs are copied to the current CUDA device and the gradients copied back. `out`: preallocated results,
    shaped as returned, written in place (for CPU inputs, after the copy back)."""
    _lib.require_cuda()
    lib = _lib.load()
    B, m, n = G.shape
    e = A.shape[1] if (A is not None and A.dim() > 1) else 0
    dtype = G.dtype
    run, home = _device_call(G.device)
    lead, R, (g,) = flatten_directions([dl_dzhat], [(B, n)], dtype, run)
    shapes = [(n, n), (n,), (m, n), (m,), (e, n), (e,), (m, m)]
    into = out is not None and home == run
    outs = [(out[k] if into else torch.empty(*lead, B, *s, dtype=dtype, device=run))
            if (need[k] and not (k in (4, 5) and e == 0)) else None for k, s in enumerate(shapes)]
    if R > 0 and B > 0:
        ins = _saved_on(run, home, e, Q, G, A, F, zhat, nu, lam, slack)
        hd = _lib.get_handle(dtype, n, m, e, run.index, torch.cuda.current_stream(run).cuda_stream)
        reuse = home == run and _reuses(saved, "struct", hd, hd.fwd_generation, B)
        flags = (1 if exact_adjoint else 0) | (2 if reuse else 0)
        with torch.cuda.device(run):
            _lib.check(lib.lcpb200_backward_batched(hd.raw, R, B, *[_lib.ptr(t) for t in ins], _lib.ptr(g),
                                                    *[_lib.ptr(t) for t in outs], None, flags, _lib.stream_ptr(run)))
    if home != run:
        outs = [None if t is None else (t.to(home) if out is None else out[k].copy_(t)) for k, t in enumerate(outs)]
    return tuple(outs)


def solve_jvp_batched(Q, G, A, F, zhat, nu, lam, slack, tangents, saved=None):
    """lcpb200_jvp_batched: tangents of (Q, p, G, h, A, b, F), each [..., *input shape] or None (zero), -> the
    tangent of zhat [..., B, n]. The leading dims, the same for every tangent, are the R directions of one call:
    each scene's KKT matrix is factored once for all of them. tQ enters as tQ zhat, as given (the backward's dQ is
    symmetrised: the two agree along symmetric tQ). CPU inputs run on the current CUDA device."""
    _lib.require_cuda()
    lib = _lib.load()
    B, m, n = G.shape
    e = A.shape[1] if (A is not None and A.dim() > 1) else 0
    dtype = G.dtype
    run, home = _device_call(G.device)
    if e == 0:
        tangents = list(tangents[:4]) + [None, None] + [tangents[6]]
    lead, R, ts = flatten_directions(tangents, [(B, n, n), (B, n), (B, m, n), (B, m), (B, e, n), (B, e), (B, m, m)],
                                     dtype, run)
    dz = torch.zeros((R, B, n), dtype=dtype, device=run)
    if R > 0 and B > 0 and any(t is not None for t in ts):
        ins = _saved_on(run, home, e, Q, G, A, F, zhat, nu, lam, slack)
        hd = _lib.get_handle(dtype, n, m, e, run.index, torch.cuda.current_stream(run).cuda_stream)
        flags = 2 if home == run and _reuses(saved, "struct", hd, hd.fwd_generation, B) else 0
        with torch.cuda.device(run):
            _lib.check(lib.lcpb200_jvp_batched(hd.raw, R, B, *[_lib.ptr(t) for t in ins], *[_lib.ptr(t) for t in ts],
                                               _lib.ptr(dz), None, flags, _lib.stream_ptr(run)))
    return dz.to(home).reshape(lead + (B, n))


def _lcp_vjp(dzhat, meta, saved):
    need, state, exact = meta
    zhat, Q, G, A, F, nu, lam, slack = saved
    if dzhat.dim() == 2:        # LCPFunction's backward: CPU inputs keep the host path and its retained state
        return solve_backward(Q, G, A, F, zhat, nu, lam, slack, dzhat, need, saved=state, exact_adjoint=exact)
    return solve_backward_batched(Q, G, A, F, zhat, nu, lam, slack, dzhat, need, saved=state, exact_adjoint=exact)


def _lcp_jvp(tangents, state, saved):
    zhat, Q, G, A, F, nu, lam, slack = saved
    return solve_jvp_batched(Q, G, A, F, zhat, nu, lam, slack, tangents, saved=state)


_BATCHED_PRIMAL = ("LCPFunction: vmap over the inputs of the solve is not supported; batch scenes along dim 0 "
                   "instead (vmap of its vector-Jacobian and Jacobian-vector products -- jacrev, jacfwd -- is supported)")
# VjpFn's meta: (need, forward's save dict, exact_adjoint); JvpFn's: the save dict. saved: _LCPFn.setup_context's.
_LCP = Solve(_lcp_vjp, _lcp_jvp, 7, "LCPFunction: second derivatives are not implemented", _BATCHED_PRIMAL,
             _BATCHED_PRIMAL)


class _LCPFn(torch.autograd.Function):
    """Written in setup_context form so that torch.func (vjp, grad, jacrev, jvp, jacfwd) and forward-mode dual
    tensors can trace through it. The primal outputs nu, lam, slack are not differentiable."""

    @staticmethod
    def forward(Q, p, G, h, A, b, F, opts):
        state = {}
        zhat, nu, lam, slack, status, iters, resid = solve_forward(
            Q, p, G, h, A, b, F, opts.eps, opts.not_improved_lim, opts.max_iter, save=state)
        if bool((status == _lib.STATUS_SINGULAR_Q).any()):
            raise RuntimeError(SINGULAR_Q_MSG)
        if opts.verbose >= 0 and bool((resid > 1.0).any()):
            print(INACCURATE_MSG)
            print(resid.max())
        opts.nus, opts.lams, opts.slacks = nu, lam, slack          # lcp.py:29 stashes these on self
        opts.status, opts.iters, opts.resids = status, iters, resid
        opts._solve_state = state                                  # picked up by setup_context, right after
        return zhat, nu, lam, slack

    @staticmethod
    def setup_context(ctx, inputs, output):
        Q, p, G, h, A, b, F, opts = inputs
        zhat, nu, lam, slack = output
        e = A.shape[1] if A.dim() > 1 else 0
        ctx.state = opts.__dict__.pop("_solve_state", None)
        ctx.exact_adjoint = bool(getattr(opts, "exact_adjoint", False))
        saved = (zhat, Q, G, A if e > 0 else None, F, nu, lam, slack)
        ctx.save_for_backward(*saved)
        ctx.save_for_forward(*saved)
        ctx.mark_non_differentiable(*[t for t in (nu, lam, slack) if t is not None])

    @staticmethod
    def backward(ctx, dl_dzhat, *_):
        need = tuple(ctx.needs_input_grad[:7])
        grads = VjpFn.apply(dl_dzhat, _LCP, (need, ctx.state, ctx.exact_adjoint), *ctx.saved_tensors)
        return (*grads, None)

    @staticmethod
    def jvp(ctx, tQ, tp, tG, th, tA, tb, tF, _):
        # the true derivative whatever exact_adjoint says: K is factored as the forward factors it
        dz = JvpFn.apply(_LCP, ctx.state, tQ, tp, tG, th, tA, tb, tF, *ctx.saved_tensors)
        return dz, None, None, None

    @staticmethod
    def vmap(info, in_dims, *args):
        raise NotImplementedError(_BATCHED_PRIMAL)


class LCPFunction:
    """A differentiable LCP solver (primal-dual interior point), H100-native.

    Mirrors `lcp_physics.lcp.lcp.LCPFunction(eps, verbose, not_improved_lim,
    max_iter)(Q, p, G, h, A, b, F)` -- reference lcp/lcp.py:12-35."""

    def __init__(self, eps=1e-12, verbose=-1, not_improved_lim=3, max_iter=10, exact_adjoint=False):
        # exact_adjoint is an extension (SURVEY.md f-4): False reproduces the reference's gradients
        self.exact_adjoint = exact_adjoint
        self.eps = eps
        self.verbose = verbose
        self.not_improved_lim = not_improved_lim
        self.max_iter = max_iter
        self.nus = self.lams = self.slacks = None
        self.status = self.iters = self.resids = None

    def __call__(self, Q, p, G, h, A, b, F):
        """zhat [B, n]. Differentiable in reverse mode (backward, torch.func.vjp / grad / jacrev, where the
        cotangents of a vmap go to one batched kernel call) and in forward mode (torch.func.jvp / jacfwd,
        torch.autograd.forward_ad dual tensors). Forward mode is the true derivative of the solve, the transpose
        of exact_adjoint=True; it takes tQ as given while the backward's dQ is symmetrised, so jacfwd and
        jacrev agree along symmetric directions of Q. Second derivatives and vmap over the inputs raise
        NotImplementedError."""
        return _LCPFn.apply(Q, p, G, h, A, b, F, self)[0]
