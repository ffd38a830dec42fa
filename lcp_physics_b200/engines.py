"""Drop-in for `lcp_physics.physics.engines.PdipmEngine` (reference physics/engines.py:17-116).

`B200PdipmEngine` exposes the same two methods the reference `World` calls --
`solve_dynamics(world, dt) -> new_v` (world.py:86) and `post_stabilization(world)`
(world.py:111) -- plus the `max_iter` / `lcp_solver` attributes, and is selected
with `World(engine=B200PdipmEngine)` (world.py:26, utils.py:142-150) without any
edit to the reference.

What moves to the GPU: the dense assembly the reference does with Python loops
over contacts (`World.Jc/Jf/E/mu/restitutions`, world.py:144-234) and with
`torch.cat`/slice assignment (engines.py:50-74) is one CUDA kernel
(`lcpb200_assemble`) fed by the stacked contact list; it is differentiable
(`lcpb200_assemble_backward`), so gradients still reach contact normals/points,
friction, restitution, masses, velocities and forces. The LCP itself is
`lcp_physics_b200.LCPFunction`. Host-side control flow (no-contact branch, joint
rows `World.Je()`, sign conventions) stays Python, like the reference.

Reads from `world` exactly what the reference engine reads (engines.py:27-77):
`t, bodies, contacts, vec_len, static_inverse, M(), Je(), apply_forces(t), get_v()`
and per-body `fric_coeff`, `restitution`; `world.fric_dirs` must be 2
(world.py:191-192 hard-codes dir2 = -dir1).
"""
import torch

from . import _lib
from ._derivatives import JvpFn, Solve, VjpFn, flatten_directions
from .lcp import LCPFunction


class Engine:
    """Base class for stepping engine (engines.py:11-14)."""

    def solve_dynamics(self, world, dt):
        raise NotImplementedError


class _AssembleFn(torch.autograd.Function):
    """(mass, inertia, v, fext, normal, p1, p2, mu, rest) -> (Q, p, G, h, F), batched [B, ...] CUDA tensors."""

    @staticmethod
    def forward(ctx, mass, inertia, v, fext, normal, p1, p2, mu, rest, body1, body2, dt):
        lib = _lib.load()
        B, nb = mass.shape
        nc = normal.shape[1]
        n, m = 3 * nb, 4 * nc
        dt_ = mass.dtype
        dev = mass.device
        ins = [t.contiguous() for t in (mass, inertia, v, fext, normal, p1, p2)]
        mu_c, rest_c = mu.contiguous(), rest.contiguous()
        new = lambda *s: torch.empty(*s, dtype=dt_, device=dev)
        Q, p, G, h, F = new(B, n, n), new(B, n), new(B, m, n), new(B, m), new(B, m, m)
        with torch.cuda.device(dev):
            _lib.check(lib.lcpb200_assemble(
                _lib.dtype_code(dt_), B, nb, nc, float(dt),
                *[_lib.ptr(t) for t in ins], _lib.ptr(body1), _lib.ptr(body2), _lib.ptr(mu_c), _lib.ptr(rest_c),
                *[_lib.ptr(t) for t in (Q, p, G, h, F)], _lib.stream_ptr(dev)))
        ctx.save_for_backward(*ins[:3], *ins[4:], mu_c, rest_c, body1, body2)
        ctx.dt = float(dt)
        ctx.dims = (B, nb, nc)
        return Q, p, G, h, F

    @staticmethod
    def backward(ctx, dQ, dp, dG, dh, dF):
        lib = _lib.load()
        mass, inertia, v, normal, p1, p2, mu, rest, body1, body2 = ctx.saved_tensors
        B, nb, nc = ctx.dims
        dt_ = mass.dtype
        dev = mass.device
        z = lambda t: torch.zeros_like(t)
        up = [g.contiguous() if g is not None else torch.zeros(s, dtype=dt_, device=dev)
              for g, s in zip((dQ, dp, dG, dh, dF),
                              ((B, 3 * nb, 3 * nb), (B, 3 * nb), (B, 4 * nc, 3 * nb), (B, 4 * nc), (B, 4 * nc, 4 * nc)))]
        outs = [z(mass), z(inertia), z(v), z(v), z(normal), z(p1), z(p2), z(mu), z(rest)]
        with torch.cuda.device(dev):
            _lib.check(lib.lcpb200_assemble_backward(
                _lib.dtype_code(dt_), B, nb, nc, ctx.dt,
                *[_lib.ptr(t) for t in (mass, inertia, v, normal, p1, p2)], _lib.ptr(body1), _lib.ptr(body2),
                _lib.ptr(mu), _lib.ptr(rest), *[_lib.ptr(t) for t in up], *[_lib.ptr(t) for t in outs],
                _lib.stream_ptr(dev)))
        dmass, dinertia, dv, dfext, dnormal, dp1, dp2, dmu, drest = outs
        return dmass, dinertia, dv, dfext, dnormal, dp1, dp2, dmu, drest, None, None, None


def assemble_contacts(mass, inertia, v, fext, normal, p1, p2, mu, rest, body1, body2, dt):
    """Differentiable contact-list -> dense LCP assembly on the GPU (world.py:144-234 + engines.py:50-74).
    Shapes: mass/inertia [B,nb], v/fext [B,3nb], normal/p1/p2 [B,nc,2], mu/rest [B,nc], body1/body2 [nc] int32."""
    _lib.require_cuda()
    return _AssembleFn.apply(mass, inertia, v, fext, normal, p1, p2, mu, rest, body1, body2, dt)


def _engine_args(meta, saved):
    """The handle for the current stream and the argument block both engine derivative entries
    (lcpb200_engine_backward_batched, lcpb200_engine_jvp_batched) take after R: B, nb, nc, mode, dt, the seven
    inputs, body1, body2, counts, mu, rest, A and the saved zhat, nu, lam, slack. Returns (handle, args, held):
    the pointers in args point into held, which must outlive the call."""
    (mass, inertia, v, fext, normal, p1, p2, mu, rest, A, body1, body2, zhat, nu, lam, slack, counts) = saved
    dt, mode, _exact, B, nb, nc, e = meta
    held = [None if t is None else t.contiguous()
            for t in (mass, inertia, v, fext, normal, p1, p2, body1, body2, counts, mu, rest, A, zhat, nu, lam, slack)]
    hd = _lib.get_handle(mass.dtype, 3 * nb, (4 if mode == 0 else 1) * nc, e, mass.device.index,
                         torch.cuda.current_stream(mass.device).cuda_stream)
    return hd, [B, nb, nc, mode, dt] + [_lib.ptr(t) for t in held], held


def _engine_backward(dzhat, meta, saved):
    """lcpb200_engine_backward_batched: dzhat [..., B, n] -> the 11 gradients (mass ... rest, A, b), each with
    dzhat's leading dims in front. The leading dims are the R cotangents of one call: each scene's KKT matrix is
    factored once for all of them."""
    _dt, _mode, exact, B, nb, _nc, e = meta
    mass = saved[0]
    dev = mass.device
    lead, R, (g,) = flatten_directions([dzhat], [(B, 3 * nb)], mass.dtype, dev)
    # saved[:10]: mass, inertia, v, fext, normal, p1, p2, mu, rest, A (None when e == 0)
    outs = [None if t is None else torch.zeros((R,) + tuple(t.shape), dtype=t.dtype, device=dev) for t in saved[:10]]
    outs.append(torch.zeros(R, B, e, dtype=mass.dtype, device=dev) if e > 0 else None)
    hd, args, held = _engine_args(meta, saved)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().lcpb200_engine_backward_batched(
            hd.raw, R, *args, _lib.ptr(g), *[_lib.ptr(t) for t in outs], 1 if exact else 0, _lib.stream_ptr(dev)))
    return tuple(None if t is None else t.reshape(lead + tuple(t.shape[1:])) for t in outs)


def _engine_jvp(tangents, meta, saved):
    """lcpb200_engine_jvp_batched: tangents of (mass, inertia, v, fext, normal, p1, p2, mu, rest, A, b), each
    [..., *input shape] or None (zero), -> the tangent of zhat [..., B, n]. The leading dims, the same for every
    tangent, are the R directions of one call: each scene's KKT matrix is factored once for all of them."""
    _dt, _mode, _exact, B, nb, _nc, e = meta
    mass = saved[0]
    dev = mass.device
    if e == 0:
        tangents = list(tangents[:9]) + [None, None]
    shapes = [t.shape for t in saved[:9]] + [(B, e, 3 * nb), (B, e)]
    lead, R, ts = flatten_directions(tangents, shapes, mass.dtype, dev)
    dz = torch.zeros((R, B, 3 * nb), dtype=mass.dtype, device=dev)
    if any(t is not None for t in ts) and R > 0:
        hd, args, held = _engine_args(meta, saved)
        with torch.cuda.device(dev):
            _lib.check(_lib.load().lcpb200_engine_jvp_batched(
                hd.raw, R, *args, *[_lib.ptr(t) for t in ts], _lib.ptr(dz), _lib.stream_ptr(dev)))
    return dz.reshape(lead + (B, 3 * nb))


# VjpFn's and JvpFn's meta: _EngineSolveFn's ctx.meta; saved: its saved tensors
_ENGINE = Solve(
    _engine_backward, _engine_jvp, 11, "engine_solve: second derivatives are not implemented",
    "engine_solve: vmap over the inputs of the solve is not supported; batch scenes along dim 0 instead (vmap of the "
    "vector-Jacobian product -- torch.func.vjp, jacrev -- is supported)",
    "engine_solve: vmap over the inputs of the solve is not supported; batch scenes along dim 0 instead (vmap of the "
    "Jacobian-vector product -- torch.func.jvp, jacfwd -- is supported)")


class _EngineSolveFn(torch.autograd.Function):
    """Fused path (lcpb200_engine_forward / _backward): contact structure-of-arrays in, LCP solution out.
    No dense Q / G / F exists anywhere; the backward returns gradients w.r.t. the contact list.
    mode 0 = solve_dynamics' LCP (engines.py:50-76), mode 1 = post_stabilization's (engines.py:80-116).
    Written in setup_context form so that torch.func.vjp / grad / jacrev can trace through it."""

    @staticmethod
    def forward(mass, inertia, v, fext, normal, p1, p2, mu, rest, A, b, body1, body2, dt, mode, max_iter, exact,
                counts=None):
        lib = _lib.load()
        B, nb = mass.shape
        nc = normal.shape[1]
        n, m = 3 * nb, (4 if mode == 0 else 1) * nc
        e = A.shape[1] if (A is not None and A.dim() > 1) else 0
        dt_, dev = mass.dtype, mass.device
        ins = [t.contiguous() for t in (mass, inertia, v, fext, normal, p1, p2)]
        mu_c, rest_c = mu.contiguous(), rest.contiguous()
        A_c = A.contiguous() if e > 0 else None
        b_c = b.contiguous() if e > 0 else None
        hd = _lib.get_handle(dt_, n, m, e, dev.index, torch.cuda.current_stream(dev).cuda_stream)
        new = lambda *s, d=dt_: torch.empty(*s, dtype=d, device=dev)
        zhat, lam, slack = new(B, n), new(B, m), new(B, m)
        nu = new(B, e) if e > 0 else None
        status, iters, resid = new(B, d=torch.int32), new(B, d=torch.int32), new(B)
        with torch.cuda.device(dev):
            _lib.check(lib.lcpb200_engine_forward(
                hd.raw, B, nb, nc, int(mode), float(dt), *[_lib.ptr(t) for t in ins], _lib.ptr(body1), _lib.ptr(body2),
                _lib.ptr(counts), _lib.ptr(mu_c), _lib.ptr(rest_c), _lib.ptr(A_c), _lib.ptr(b_c), 1e-12, 3, int(max_iter),
                *[_lib.ptr(t) for t in (zhat, nu, lam, slack, status, iters, resid)], _lib.stream_ptr(dev)))
        _last_info.update(iters=iters, resid=resid, status=status, lam=lam, slack=slack, nu=nu)
        return zhat, status, nu, lam, slack

    @staticmethod
    def setup_context(ctx, inputs, output):
        (mass, inertia, v, fext, normal, p1, p2, mu, rest, A, b, body1, body2, dt, mode, max_iter, exact) = inputs[:17]
        counts = inputs[17] if len(inputs) > 17 else None
        zhat, status, nu, lam, slack = output
        B, nb = mass.shape
        e = A.shape[1] if (A is not None and A.dim() > 1) else 0
        saved = (mass, inertia, v, fext, normal, p1, p2, mu, rest, A if e > 0 else None, body1, body2, zhat, nu, lam,
                 slack, counts)
        ctx.save_for_backward(*saved)
        ctx.save_for_forward(*saved)
        ctx.meta = (float(dt), int(mode), bool(exact), B, nb, normal.shape[1], e)
        ctx.mark_non_differentiable(*[t for t in (status, nu, lam, slack) if t is not None])

    @staticmethod
    def backward(ctx, dzhat, *_):
        grads = VjpFn.apply(dzhat, _ENGINE, ctx.meta, *ctx.saved_tensors)
        return (*grads, None, None, None, None, None, None, None)

    @staticmethod
    def jvp(ctx, *tangents):
        # the true derivative whatever exact_adjoint says: K is factored as the forward factors it
        dzhat = JvpFn.apply(_ENGINE, ctx.meta, *tangents[:_ENGINE.n_tangents], *ctx.saved_tensors)
        return dzhat, None, None, None, None

    @staticmethod
    def vmap(info, in_dims, *args):
        raise NotImplementedError(
            "engine_solve: vmap over the inputs of the solve is not supported; batch scenes along dim 0 instead")


_last_info = {}


def last_solve_info():
    """Diagnostics of the most recent engine_solve call (device tensors): PDIPM iteration counts, best residuals,
    status, multipliers, slacks and equality multipliers (nu, None without equality rows) per scene (the reference
    prints them with verbose >= 1, pdipm.py:97-105)."""
    return _last_info


def engine_solve(mass, inertia, v, fext, normal, p1, p2, mu, rest, body1, body2, dt, A=None, b=None, mode=0,
                 max_iter=10, exact_adjoint=False, counts=None):
    """Batched, differentiable LCP of the engine straight from the contact list (CUDA tensors):
    mass/inertia [B,nb], v/fext [B,3nb], normal/p1/p2 [B,nc,2], mu/rest [B,nc], body1/body2 [nc] int32,
    optional equality rows A [B,e,3nb], b [B,e]. Returns (zhat [B,3nb], status [B]); status == -100 marks a
    scene whose topology the fused kernel does not take (use assemble_contacts + LCPFunction for it).
    solve_dynamics: new_v = -zhat (engines.py:76); post_stabilization: dp = -zhat (engines.py:116).
    counts [B] int32 (batched worlds): scene s uses its first counts[s] contacts; body1/body2 are then [B,nc].
    body2 >= nb names a static obstacle (no dofs: a wall, floor or ramp): a one-body contact whose rows touch body1's
    three columns only -- the reference's formulation with the obstacle pinned by a TotalConstraint, reduced by the
    pinned dofs; its p2 is unused (zero gradient). body1 must be a body (< nb).
    Differentiable in reverse mode (backward, torch.func.vjp / grad / jacrev) and in forward mode (torch.func.jvp /
    jacfwd, torch.autograd.forward_ad dual tensors); the k directions of a jacfwd or vmap(jvp) go to one kernel call.
    Forward mode is always the true derivative of the solve, the transpose of the exact_adjoint=True backward; with
    exact_adjoint=False the backward gives the reference's gradients, so jacfwd and jacrev then differ whenever
    friction is on (DESIGN.md section 3.4). Second derivatives are not implemented."""
    _lib.require_cuda()
    zhat, status = _EngineSolveFn.apply(mass, inertia, v, fext, normal, p1, p2, mu, rest, A, b, body1, body2, dt, mode,
                                        max_iter, exact_adjoint, counts)[:2]
    return zhat, status


class B200PdipmEngine(Engine):
    """Engine that solves the contact LCP with the CUDA PDIPM kernels (mirror of engines.py:17-116)."""

    def __init__(self, max_iter=10, fused=True, exact_adjoint=False):
        # fused: contact list -> solution in one kernel (lcpb200_engine_forward); False (or an unsupported
        # topology / size) assembles the dense LCP on the GPU and calls LCPFunction, like the reference.
        # exact_adjoint: gradients through the transposed KKT system (the true adjoint, DESIGN.md section 3.4)
        # on both paths; False reproduces the reference's gradients, which are biased whenever friction is on.
        self.fused = fused
        self.lcp_solver = LCPFunction
        self.cached_inverse = None
        self.max_iter = max_iter
        self.exact_adjoint = exact_adjoint

    def _dense_solver(self, **kw):
        """`self.lcp_solver(**kw)`, with exact_adjoint passed on; a replaced solver cannot honour it."""
        if not self.exact_adjoint:
            return self.lcp_solver(**kw)
        if self.lcp_solver is not LCPFunction:
            raise ValueError("B200PdipmEngine(exact_adjoint=True) needs lcp_solver = lcp_physics_b200.LCPFunction; "
                             "%r would return the reference's gradients" % (self.lcp_solver,))
        return self.lcp_solver(exact_adjoint=True, **kw)

    # ------------------------------------------------------------------ helpers
    @staticmethod
    def _device():
        _lib.require_cuda()
        return torch.device("cuda", torch.cuda.current_device())

    @staticmethod
    def _contact_soa(world, dev):
        """Stack `world.contacts` ([((normal, p1, p2, pen), i1, i2)], contacts.py:203-204) into SoA tensors."""
        if getattr(world, "fric_dirs", 2) != 2:
            raise NotImplementedError("B200PdipmEngine supports fric_dirs == 2 (world.py:191-192)")
        cs = world.contacts
        normal = torch.stack([c[0][0] for c in cs]).unsqueeze(0)
        p1 = torch.stack([c[0][1] for c in cs]).unsqueeze(0)
        p2 = torch.stack([c[0][2] for c in cs]).unsqueeze(0)
        b1 = torch.tensor([c[1] for c in cs], dtype=torch.int32, device=dev)
        b2 = torch.tensor([c[2] for c in cs], dtype=torch.int32, device=dev)
        bodies = world.bodies
        base = normal
        as_t = lambda x: x if isinstance(x, torch.Tensor) else base.new_tensor(x)
        mu = torch.stack([0.5 * (as_t(bodies[c[1]].fric_coeff) + as_t(bodies[c[2]].fric_coeff)).reshape(())
                          for c in cs]).unsqueeze(0)                                  # world.py:213-224
        rest = torch.stack([0.5 * (as_t(bodies[c[1]].restitution) + as_t(bodies[c[2]].restitution)).reshape(())
                            for c in cs]).unsqueeze(0)                                # world.py:144-151
        return normal.to(dev), p1.to(dev), p2.to(dev), b1, b2, mu.to(dev), rest.to(dev)

    def _assemble(self, world, dt, fext, dev):
        M = world.M()
        v = world.get_v()
        n = M.size(0)
        Md = torch.diagonal(M)
        if bool((M - torch.diag(Md)).abs().max() != 0):
            raise NotImplementedError("B200PdipmEngine expects the block-diagonal mass matrix of world.py:57-61 "
                                      "to be diagonal ([I, m, m] per body, bodies.py:44-47)")
        vlen = world.vec_len
        if vlen != 3:
            raise NotImplementedError("2-D bodies (vec_len == 3) only")
        Mb = Md.reshape(-1, 3)
        inertia, mass = Mb[:, 0].unsqueeze(0), Mb[:, 1].unsqueeze(0)
        normal, p1, p2, b1, b2, mu, rest = self._contact_soa(world, dev)
        return assemble_contacts(mass.to(dev), inertia.to(dev), v.unsqueeze(0).to(dev), fext.unsqueeze(0).to(dev),
                                 normal, p1, p2, mu, rest, b1, b2, dt), n

    def _fused(self, world, dt, fext, Je, ge, dev, mode, max_iter):
        """One lcpb200_engine_forward call for this world (batch of one); None when the fused kernel cannot
        take it (non-diagonal M, vec_len != 3, unsupported topology, a large scene that is not float64)."""
        M = world.M()
        Md = torch.diagonal(M)
        neq = Je.size(0) if Je.ndimension() > 0 else 0
        if world.vec_len != 3:
            return None
        if M.size(0) + neq > 128 or len(world.contacts) * 4 > 1024:
            # large scene: banded kernel (fp64, <= 16 border rows); otherwise the dense path
            if M.dtype != torch.float64 or neq > 16:
                return None
        if bool((M - torch.diag(Md)).abs().max() != 0):
            return None
        Mb = Md.reshape(-1, 3)
        normal, p1, p2, b1, b2, mu, rest = self._contact_soa(world, dev)
        v = world.get_v()
        if neq > 0:
            A = Je.unsqueeze(0).to(dev)
            b = (ge.unsqueeze(0).to(dev) if ge is not None else A.new_zeros(1, neq))
        else:
            A = b = None
        x, status = engine_solve(Mb[:, 1].unsqueeze(0).to(dev), Mb[:, 0].unsqueeze(0).to(dev), v.unsqueeze(0).to(dev),
                                 fext.unsqueeze(0).to(dev), normal, p1, p2, mu, rest, b1, b2, dt, A=A, b=b, mode=mode,
                                 max_iter=max_iter, exact_adjoint=self.exact_adjoint)
        st = int(status[0])
        if st == _lib.STATUS_SINGULAR_Q:
            from .lcp import SINGULAR_Q_MSG
            raise RuntimeError(SINGULAR_Q_MSG)
        return None if st == -100 else x

    # ------------------------------------------------------------------ engines.py:26-78
    def solve_dynamics(self, world, dt):
        t = world.t
        Je = world.Je()
        neq = Je.size(0) if Je.ndimension() > 0 else 0

        f = world.apply_forces(t)
        v0 = world.get_v()
        if not world.contacts:
            # no contact constraints, no complementarity (engines.py:35-49): host-side dense solve
            u = torch.matmul(world.M(), v0) + dt * f
            if neq > 0:
                u = torch.cat([u, u.new_zeros(neq)])
                P = torch.cat([torch.cat([world.M(), -Je.t()], dim=1),
                               torch.cat([Je, Je.new_zeros(neq, neq)], dim=1)])
            else:
                P = world.M()
            if self.cached_inverse is None:
                inv = torch.inverse(P)
                if world.static_inverse:
                    self.cached_inverse = inv
            else:
                inv = self.cached_inverse
            x = torch.matmul(inv, u)
            return x[:world.vec_len * len(world.bodies)]
        dev = self._device()
        if self.fused and self.lcp_solver is LCPFunction:
            x = self._fused(world, dt, f, Je, None, dev, mode=0, max_iter=self.max_iter)
            if x is not None:
                return (-x).squeeze(0).to(v0.device)                  # engines.py:76
        (Q, p, G, h, F), n = self._assemble(world, dt, f, dev)
        if neq > 0:
            A = Je.unsqueeze(0).to(dev)
            b = A.new_zeros(1, neq)
        else:
            A = torch.tensor([], dtype=Q.dtype, device=dev)       # engines.py:59-60
            b = torch.tensor([], dtype=Q.dtype, device=dev)
        x = -self._dense_solver(max_iter=self.max_iter, verbose=-1)(Q, p, G, h, A, b, F)   # engines.py:76
        new_v = x[:, :world.vec_len * len(world.bodies)].squeeze(0)
        return new_v.to(v0.device)

    # ------------------------------------------------------------------ engines.py:80-116
    def post_stabilization(self, world):
        v = world.get_v()
        M = world.M()
        Je = world.Je()
        ge = torch.matmul(Je, v)
        if not world.contacts:
            u = torch.cat([Je.new_zeros(Je.size(1)), ge])
            neq = Je.size(0) if Je.ndimension() > 0 else 0
            if neq > 0:
                P = torch.cat([torch.cat([M, -Je.t()], dim=1), torch.cat([Je, Je.new_zeros(neq, neq)], dim=1)])
            else:
                P = M
            inv = torch.inverse(P) if self.cached_inverse is None else self.cached_inverse
            x = torch.matmul(inv, u)
            return -x[:M.size(0)]
        dev = self._device()
        fzero = v.new_zeros(v.shape)
        if self.fused and self.lcp_solver is LCPFunction:
            x = self._fused(world, 0.0, fzero, Je, ge, dev, mode=1, max_iter=10)      # engines.py:114: default max_iter
            if x is not None:
                return (-x).to(v.device)
        (Q, _p, G, _h, _F), n = self._assemble(world, 0.0, fzero, dev)
        nc = len(world.contacts)
        Jc = G[:, :nc, :]
        _, _, _, _, _, _, rest = self._contact_soa(world, dev)
        jv = torch.bmm(Jc, v.unsqueeze(0).unsqueeze(2).to(dev)).squeeze(2)
        gc = jv + jv * -rest                                       # engines.py:90
        hvec = Q.new_zeros(1, n)
        if Je.ndimension() > 0 and Je.size(0) > 0:
            A = Je.unsqueeze(0).to(dev)
            b = ge.unsqueeze(0).to(dev)
        else:
            A = torch.tensor([], dtype=Q.dtype, device=dev)
            b = torch.tensor([], dtype=Q.dtype, device=dev)
        Fz = Q.new_zeros(1, nc, nc)
        x = self._dense_solver()(Q, hvec, Jc.contiguous(), gc, A, b, Fz)   # engines.py:114 (default max_iter)
        return (-x).to(v.device)                                   # [1, n]; the caller squeezes (world.py:111)
