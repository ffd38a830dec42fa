"""GPU: the banded large-scene kernel (csrc/lcp_banded.cuh) at its band and border limits, fp64, `engine_solve`.

* Mirror check: for every scene the kernel's own half bandwidth bw (the sum the forward adds to the profile
  counter `c_gradients`, batch of one, read before any backward) equals the host restatement's
  (tests/band_plan.py).
* The widest supported bands: bwa = 128 against the condensed kernel and against the CPU oracle (Wc >= Nbp
  included), and the maximum of a lower tier (bwa = 120 at 779 bodies): a relabelling of the bodies agrees, and
  an fp64 KKT residual recomputed on the host from the contact list reproduces the kernel's best residual.
* One step past the limit, in each of the four ranges where the leftover shared memory held a window one tier
  wider than the plan's band storage (A: 44-58 bodies, B: 774-812, C: 1493-1530, D: 2174-2210) and past the
  window itself: status -100, zero gradients, the other scenes of the batch bitwise unchanged, and
  `B200PdipmEngine` falls back to its dense path.
* The border: 16 rows solved, 17 rejected; degree 12 in the band, 13 in the border, one-body contacts not
  counted; hub-hub contacts; hubs with > 32 and > 256 contacts; an empty band and a band of one body.
* Topology: components, isolated bodies and bodies that touch only obstacles; every residue of Nb mod 8; a
  zero-contact scene inside a banded batch; pairs with two contacts.

Reference: `pdipm_oracle.lcp_forward(coupled=False)` on the plain-torch dense assembly below (one-body contacts,
arbitrary A), gradients from `lcp_backward_from_saved` / `lcp_backward_exact_from_saved` fed the kernel's
forward state and chained to the contact list by autograd through that assembly. fp64 contracts (DESIGN.md
section 5): forward 1e-6, gradients 1e-4.
"""
import os

import numpy as np
import pytest
import torch

from tests import band_plan as bp

pytestmark = pytest.mark.gpu
NAMES = ["mass", "inertia", "v", "fext", "normal", "p1", "p2", "mu", "restitution"]
DT = 1.0 / 30
f64 = torch.float64


@pytest.fixture
def forced_banded():
    from lcp_physics_b200 import _lib

    def set_(on):
        if on:
            os.environ["LCPB200_FORCE_BANDED"] = "1"
        else:
            os.environ.pop("LCPB200_FORCE_BANDED", None)
        _lib.clear_handles()
    yield set_
    set_(False)


# ------------------------------------------------------------------------------------------ dense reference
def _cross(a, b):
    return a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]


def dense_lcp(t, mode, dt=DT):
    """(Q, p, G, h, A, b, F) of the engine's LCP from the contact list t (CPU tensors, body lists [nc]):
    mode 0 = solve_dynamics (engines.py:50-76), mode 1 = post_stabilization (engines.py:80-116). body2 >= nb is a
    static obstacle: its contact rows touch body1's columns only."""
    mass, inertia, v, fext = t["mass"], t["inertia"], t["v"], t["fext"]
    normal, p1, p2, mu, rest = t["normal"], t["p1"], t["p2"], t["mu"], t["restitution"]
    b1, b2 = t["body1"].long(), t["body2"].long()
    B, nb = mass.shape
    nc, n = normal.shape[1], 3 * nb
    ar = torch.arange(nc)
    S1 = torch.zeros(nc, nb + 1, dtype=f64)
    S1[ar, b1] = 1
    S2 = torch.zeros(nc, nb + 1, dtype=f64)
    S2[ar, b2.clamp(max=nb)] = 1
    S1, S2 = S1[:, :nb], S2[:, :nb]                     # the obstacle column is dropped

    def rows(d):
        r1 = torch.stack([_cross(p1, d), d[..., 0], d[..., 1]], -1)
        r2 = -torch.stack([_cross(p2, d), d[..., 0], d[..., 1]], -1)
        return (S1[None, :, :, None] * r1[:, :, None, :] + S2[None, :, :, None] * r2[:, :, None, :]).reshape(B, nc, n)

    Md = torch.stack([inertia, mass, mass], -1).reshape(B, n)
    Q = torch.diag_embed(Md)
    Jc = rows(normal)
    jv = torch.bmm(Jc, v.unsqueeze(2)).squeeze(2)
    if mode == 0:
        d1 = torch.stack([normal[..., 1], -normal[..., 0]], -1)
        Jf = torch.stack([rows(d1), rows(-d1)], 2).reshape(B, 2 * nc, n)
        G = torch.cat([Jc, Jf, torch.zeros(B, nc, n, dtype=f64)], 1)
        E = torch.zeros(2 * nc, nc, dtype=f64)
        E[2 * ar, ar] = 1
        E[2 * ar + 1, ar] = 1
        F = torch.zeros(B, 4 * nc, 4 * nc, dtype=f64)
        F[:, nc:3 * nc, 3 * nc:] = E
        F[:, 3 * nc:, :nc] = torch.diag_embed(mu)
        F[:, 3 * nc:, nc:3 * nc] = -E.t()
        p = Md * v + dt * fext
        h = torch.cat([jv * rest, torch.zeros(B, 3 * nc, dtype=f64)], 1)
    else:
        G, F = Jc, torch.zeros(B, nc, nc, dtype=f64)
        p = torch.zeros(B, n, dtype=f64)
        h = jv + jv * -rest
    if t.get("A") is not None:
        A, b = t["A"], t["b"]
    else:
        A = b = torch.tensor([], dtype=f64)
    return Q, p, G, h, A, b, F


def oracle(t, mode, max_iter=10):
    from oracle import pdipm_oracle as po
    with torch.no_grad():
        return po.lcp_forward(*dense_lcp(t, mode), max_iter=max_iter, coupled=False)


def oracle_grads(t, mode, k, gz, exact):
    """Gradients w.r.t. the contact list of sum(zhat * gz), from the kernel's saved forward state k."""
    from oracle import pdipm_oracle as po
    keys = NAMES + (["A", "b"] if t.get("A") is not None else [])
    leaves = {name: t[name].clone().requires_grad_(True) for name in keys}
    inp = dense_lcp(dict(t, **leaves), mode)
    fn = po.lcp_backward_exact_from_saved if exact else po.lcp_backward_from_saved
    d = fn(tuple(x.detach() for x in inp), k["z"], k["nu"], k["lam"], k["slack"], gz)
    outs = [(x, g) for x, g in zip(inp, d) if g is not None and x.requires_grad]
    torch.autograd.backward([x for x, _ in outs], [g for _, g in outs])
    return {name: (leaves[name].grad if leaves[name].grad is not None else torch.zeros_like(leaves[name]))
            for name in keys}


# ------------------------------------------------------------------------------------------ kernel
def solve(t, mode, gz=None, exact=False, counts=None, max_iter=10):
    """engine_solve on the GPU; returns CPU tensors z, status, resid, iters, lam, slack, nu and, given gz, the
    gradients of sum(z * gz)."""
    from lcp_physics_b200.engines import engine_solve, last_solve_info
    keys = NAMES + (["A", "b"] if t.get("A") is not None else [])
    leaves = {name: t[name].cuda().clone().requires_grad_(gz is not None) for name in keys}
    B = t["mass"].shape[0]
    b1, b2 = t["body1"].cuda(), t["body2"].cuda()
    if counts is not None:
        b1, b2 = (x.unsqueeze(0).expand(B, -1).contiguous() if x.dim() == 1 else x for x in (b1, b2))
        counts = torch.as_tensor(counts, dtype=torch.int32).cuda()
    z, st = engine_solve(*[leaves[k] for k in NAMES], b1, b2, DT, A=leaves.get("A"), b=leaves.get("b"), mode=mode,
                         max_iter=max_iter, exact_adjoint=exact, counts=counts)
    info = last_solve_info()
    out = dict(z=z.detach().cpu(), status=st.cpu(), resid=info["resid"].cpu(), iters=info["iters"].cpu(),
               lam=info["lam"].cpu(), slack=info["slack"].cpu(), nu=None if info["nu"] is None else info["nu"].cpu())
    if gz is not None:
        (z * gz.cuda()).sum().backward()
        out["grads"] = {k: (v.grad.cpu() if v.grad is not None else torch.zeros(v.shape, dtype=f64))
                        for k, v in leaves.items()}
    torch.cuda.synchronize()
    return out


def kernel_bw(t, mode):
    """The kernel's half bandwidth bw of a batch-of-one scene (0 when the scene is rejected)."""
    from lcp_physics_b200 import _lib
    nb, nc = t["mass"].shape[1], t["normal"].shape[1]
    e = t["A"].shape[1] if t.get("A") is not None else 0
    hd = _lib.get_handle(f64, 3 * nb, (4 if mode == 0 else 1) * nc, e, torch.cuda.current_device(),
                         torch.cuda.current_stream().cuda_stream)
    hd.profile(True)
    with torch.no_grad():
        solve(t, mode)
    prof = hd.profile(False)
    return prof["c_gradients"]


def rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def grad_errs(got, ref):
    """Per-leaf relative errors; a leaf whose reference gradient is round-off (below 1e-9 of the largest one: the
    inertia in post-stabilisation, where midpoint contacts carry no torque) is measured against that scale."""
    scale = max(float(g.norm()) for g in ref.values())
    errs = {}
    for name, g in ref.items():
        assert torch.isfinite(got[name]).all(), name
        errs[name] = float((got[name] - g).norm()) / max(float(g.norm()), 1e-9 * scale, 1e-300)
    return errs


def check_oracle(t, mode, sc_order, exacts=(False,), fwd_tol=1e-6, max_iter=10):
    """Mirror check, forward against the oracle, gradients against the oracle's through the dense assembly."""
    assert kernel_bw(t, mode) == sc_order["bw"]
    gz = torch.randn(t["v"].shape, generator=torch.Generator().manual_seed(5), dtype=f64)
    ref = oracle(t, mode, max_iter=max_iter)
    errs = {}
    for exact in exacts:
        k = solve(t, mode, gz=gz, exact=exact, max_iter=max_iter)
        assert (k["status"] >= 0).all(), k["status"].tolist()
        errs["z"] = rel(k["z"], ref.zhat)
        assert errs["z"] < fwd_tol, errs
        ge = grad_errs(k["grads"], oracle_grads(t, mode, k, gz, exact))
        errs.update({(name, exact): v for name, v in ge.items()})
        assert max(ge.values()) < 1e-4, errs
    return errs


def scene_inputs(sc, B=1, seed=0, **kw):
    return bp.to_soa(sc, B=B, seed=seed, **kw)


# ------------------------------------------------------------------------------------------ widest bands
def test_widest_band_matches_condensed(forced_banded):
    """nb = 42 at bwb = 40: bwa = 128 with n = 126, so the condensed kernel takes the same scene in post-stabilisation
    (m = 251). In mode 0 (m = 1004) the condensed plan does not fit shared memory and both calls would reach the
    banded kernel, so the forced banded kernel is checked against the oracle there."""
    sc = bp.random_graph(42, 40, mean_deg=12.0)
    o = bp.order_scene(sc)
    assert o["bwa"] == 128
    t = scene_inputs(sc, seed=1)
    gz = torch.randn(t["v"].shape, generator=torch.Generator().manual_seed(1), dtype=f64)
    res = {}
    for force in (False, True):
        forced_banded(force)
        # the condensed forward adds nothing to the counter the banded forward adds bw to
        assert kernel_bw(t, 1) == (o["bw"] if force else 0)
        res[force] = solve(t, 1, gz=gz)
        assert (res[force]["status"] >= 0).all()
    c, b = res[False], res[True]
    assert rel(b["z"], c["z"]) < 1e-8, rel(b["z"], c["z"])
    errs = grad_errs(b["grads"], c["grads"])
    assert max(errs.values()) < 1e-4, errs
    check_oracle(scene_inputs(sc, seed=0), 0, o, exacts=(False, True))


@pytest.mark.parametrize("key", [(44, 17, 12.0), (45, 1, 12.0), (50, 3, 8.0), (58, 4, 6.0)])
@pytest.mark.parametrize("mode", [0, 1])
def test_wide_bands_match_oracle(key, mode):
    """bwb 41-42 (bwa = 128) at 44-58 bodies; at 44 and 45 bodies the window (Wc = 136) spans the whole matrix."""
    sc = bp.random_graph(key[0], key[1], mean_deg=key[2])
    o = bp.order_scene(sc)
    assert o["bwb"] == bp.WIDE_GRAPHS[key] and o["bwa"] == 128
    t = scene_inputs(sc, seed=3)
    check_oracle(t, mode, o, exacts=(False, True) if mode == 0 else (False,))


def _kkt_resid_host(t, mode, k):
    """PDIPM residual (pdipm.py:82-96) of the kernel's returned best iterate, recomputed in fp64 with scipy.sparse
    from the contact list."""
    import scipy.sparse as sp
    nb, nc = t["mass"].shape[1], t["normal"].shape[1]
    n = 3 * nb
    b1, b2 = t["body1"].numpy().astype(np.int64), t["body2"].numpy().astype(np.int64)
    nrm, p1, p2 = t["normal"][0].numpy(), t["p1"][0].numpy(), t["p2"][0].numpy()
    v = t["v"][0].numpy()

    def rows(d):
        c1 = p1[:, 0] * d[:, 1] - p1[:, 1] * d[:, 0]
        c2 = p2[:, 0] * d[:, 1] - p2[:, 1] * d[:, 0]
        r = np.repeat(np.arange(nc), 6)
        c = np.stack([3 * b1, 3 * b1 + 1, 3 * b1 + 2, 3 * b2, 3 * b2 + 1, 3 * b2 + 2], 1).reshape(-1)
        val = np.stack([c1, d[:, 0], d[:, 1], -c2, -d[:, 0], -d[:, 1]], 1).reshape(-1)
        keep = c < n
        return sp.csr_matrix((val[keep], (r[keep], c[keep])), shape=(nc, n))

    Jc = rows(nrm)
    Md = torch.stack([t["inertia"][0], t["mass"][0], t["mass"][0]], -1).reshape(-1).numpy()
    rest = t["restitution"][0].numpy()
    jv = Jc @ v
    if mode == 0:
        d1 = np.stack([nrm[:, 1], -nrm[:, 0]], 1)
        J1, J2 = rows(d1), rows(-d1)
        Jf = sp.vstack([J1, J2]).tocsr()[np.stack([np.arange(nc), nc + np.arange(nc)], 1).reshape(-1)]
        G = sp.vstack([Jc, Jf, sp.csr_matrix((nc, n))]).tocsr()
        mu = t["mu"][0].numpy()
        ar = np.arange(nc)
        E = sp.csr_matrix((np.ones(2 * nc), (np.concatenate([2 * ar, 2 * ar + 1]), np.concatenate([ar, ar]))),
                          shape=(2 * nc, nc))
        F = sp.bmat([[sp.csr_matrix((nc, nc)), sp.csr_matrix((nc, 2 * nc)), sp.csr_matrix((nc, nc))],
                     [sp.csr_matrix((2 * nc, nc)), sp.csr_matrix((2 * nc, 2 * nc)), E],
                     [sp.diags(mu), -E.T, sp.csr_matrix((nc, nc))]], format="csr")
        p = Md * v + DT * t["fext"][0].numpy()
        h = np.concatenate([jv * rest, np.zeros(3 * nc)])
    else:
        G, F = Jc, sp.csr_matrix((nc, nc))
        p = np.zeros(n)
        h = jv + jv * -rest
    x, z, s = k["z"][0].numpy(), k["lam"][0].numpy(), k["slack"][0].numpy()
    m = z.shape[0]
    rx = G.T @ z + Md * x + p
    rz = G @ x + s - h - F @ z
    return np.linalg.norm(rz) + np.linalg.norm(rx) + m * abs(float(s @ z) / m)


@pytest.mark.parametrize("mode", [0, 1])
def test_lower_tier_maximum(mode):
    """A 41 x 19 six-family lattice: bwb 38, bwa 120 = the plan's maximum at 779 bodies."""
    sc = bp.lattice(41, 19, bp.SIX)
    o = bp.order_scene(sc)
    assert (o["bwa"], bp.carve_plan(sc["nb"], len(sc["body1"]), 4 if mode == 0 else 1)["bwa_max"]) == (120, 120)
    t = scene_inputs(sc, seed=7)
    assert kernel_bw(t, mode) == o["bw"]
    k = solve(t, mode, max_iter=5)                             # not converged: a residual well above round-off
    assert int(k["status"][0]) >= 0
    host = _kkt_resid_host(t, mode, k)
    assert abs(host - float(k["resid"][0])) <= 1e-9 * host + 1e-12, (host, float(k["resid"][0]))
    # relabel the bodies: the same LCP, the same solution
    nb = sc["nb"]
    perm = np.random.default_rng(3).permutation(nb)             # old body i -> new body perm[i]
    inv = np.argsort(perm)
    sc2 = dict(sc, pos=sc["pos"][inv], body1=perm[sc["body1"]].astype(np.int32), body2=perm[sc["body2"]].astype(np.int32))
    o2 = bp.order_scene(sc2)
    assert o2["bw"] == o["bw"]
    t2 = dict(t)
    t2["body1"], t2["body2"] = torch.from_numpy(sc2["body1"]), torch.from_numpy(sc2["body2"])
    for name in ("mass", "inertia"):
        t2[name] = t[name][:, inv]
    for name in ("v", "fext"):
        t2[name] = t[name].reshape(1, nb, 3)[:, inv].reshape(1, -1)
    assert kernel_bw(t2, mode) == o2["bw"]
    k2 = solve(t2, mode, max_iter=5)
    z2 = k2["z"].reshape(1, nb, 3)[:, perm].reshape(1, -1)
    assert rel(z2, k["z"]) < 1e-8, rel(z2, k["z"])


# ------------------------------------------------------------------------------------------ past the limit
def _window_scene(name):
    """(scene, mode, admitted partner contact count): a scene past the plan and a prefix of its contact list that
    the plan admits."""
    if name.startswith("graph"):
        nb, seed, md = {"graphA50": (50, 0, 12.0), "graphA58": (58, 6, 8.0), "graph45": (50, 5, 12.0)}[name]
        return bp.random_graph(nb, seed, mean_deg=md), 0
    return {"latticeB": (bp.lattice(40, 20, bp.FIVE), 1), "hexC": (bp.hex_pile(40, 38), 1),
            "latticeD": (bp.lattice(122, 18, ((1, 0), (0, 1), (2, 0))), 1)}[name]


@pytest.mark.parametrize("name", ["graphA50", "graphA58", "graph45", "latticeB", "hexC", "latticeD"])
def test_past_the_limit_is_rejected(name):
    sc, mode = _window_scene(name)
    nb, nc = sc["nb"], len(sc["body1"])
    o = bp.order_scene(sc)
    plan = bp.carve_plan(nb, nc, 4 if mode == 0 else 1)
    assert not bp.admitted(plan, o["bwb"], o["nbd"])
    assert bp.admitted(plan, o["bwb"], o["nbd"], old=True) == (name != "graph45")
    half = nc // 2
    oh = bp.order(nb, sc["body1"][:half], sc["body2"][:half], sc["p1"][:half], sc["p2"][:half], sc.get("A"))
    assert bp.admitted(plan, oh["bwb"], oh["nbd"]), oh["bwb"]
    t1 = scene_inputs(sc, B=1, seed=2)
    assert kernel_bw(t1, mode) == 0                             # rejected scenes add nothing
    gz1 = torch.randn(t1["v"].shape, generator=torch.Generator().manual_seed(4), dtype=f64)
    k = solve(t1, mode, gz=gz1)
    assert int(k["status"][0]) == -100 and int(k["iters"][0]) == 0 and bool(torch.isnan(k["resid"][0]))
    for g in k["grads"].values():
        assert float(g.abs().max()) == 0.0
    # in a batch: the rejected scene changes nothing for the others
    t3 = scene_inputs(sc, B=3, seed=2)
    gz3 = torch.randn(t3["v"].shape, generator=torch.Generator().manual_seed(4), dtype=f64)
    counts = [half, nc, half - 7]
    oh2 = bp.order(nb, sc["body1"][:half - 7], sc["body2"][:half - 7], sc["p1"][:half - 7], sc["p2"][:half - 7],
                   sc.get("A"))
    assert bp.admitted(plan, oh2["bwb"], oh2["nbd"]), oh2["bwb"]
    k3 = solve(t3, mode, gz=gz3, counts=counts)
    # (a rejected scene's zhat is not written: only its status and its zero gradients are defined)
    assert int(k3["status"][1]) == -100 and int(k3["status"][0]) >= 0 and int(k3["status"][2]) >= 0
    keep = [0, 2]
    t2 = {kk: (v[keep].contiguous() if torch.is_tensor(v) and v.dim() > 1 else v) for kk, v in t3.items()}
    k2 = solve(t2, mode, gz=gz3[keep], counts=[counts[0], counts[2]])
    assert torch.equal(k2["status"], k3["status"][keep])
    assert torch.equal(k2["z"], k3["z"][keep])
    for name_, g in k3["grads"].items():
        assert float(g[1].abs().max()) == 0.0, name_
        assert torch.equal(k2["grads"][name_], g[keep]), name_


def test_engine_falls_back_to_dense_path():
    """Window A through B200PdipmEngine: the fused kernel rejects the scene (status -100), the engine assembles the
    dense LCP and solves it; the result matches the oracle."""
    from lcp_physics_b200.engines import B200PdipmEngine
    from tests.helpers import ReplayWorld
    sc = bp.random_graph(50, 0, mean_deg=12.0)
    nb, nc = sc["nb"], len(sc["body1"])
    g = np.random.default_rng(9)
    fric, rest = g.uniform(0.1, 0.9, nb), g.uniform(0.2, 0.7, nb)
    t = scene_inputs(sc, seed=4)
    t["mu"] = torch.from_numpy(0.5 * (fric[sc["body1"]] + fric[sc["body2"]])).unsqueeze(0)
    t["restitution"] = torch.from_numpy(0.5 * (rest[sc["body1"]] + rest[sc["body2"]])).unsqueeze(0)
    assert int(solve(t, 0)["status"][0]) == -100
    Md = torch.stack([t["inertia"][0], t["mass"][0], t["mass"][0]], -1).reshape(-1)
    rec = dict(t=0.0, M=torch.diag(Md).numpy(), Je=np.zeros(0), v=t["v"][0].numpy(), f=t["fext"][0].numpy(),
               fric=fric, rest=rest, normal=sc["normal"], p1=sc["p1"], p2=sc["p2"], b1=sc["body1"], b2=sc["body2"])
    new_v = B200PdipmEngine(max_iter=10).solve_dynamics(ReplayWorld(rec), DT)
    ref = oracle(t, 0)
    assert rel(new_v.detach().cpu().reshape(1, -1), -ref.zhat) < 1e-6


# ------------------------------------------------------------------------------------------ border
def _pin_rows(nb, dofs):
    A = np.zeros((len(dofs), 3 * nb))
    for r, j in enumerate(dofs):
        A[r, j] = 1.0
    return A


def _with_rows(sc, A):
    sc = dict(sc)
    sc["A"] = A
    return sc


def _border_scene(name):
    if name == "border16":                  # 5 hubs of 13 contacts + 1 row on a hub: 3 x 5 + 1 = 16
        sc = bp.hubs(5, 13, ring=60)
        return _with_rows(sc, _pin_rows(sc["nb"], [1])), 16
    if name == "border17":                  # ... + 2 rows: 17
        sc = bp.hubs(5, 13, ring=60)
        return _with_rows(sc, _pin_rows(sc["nb"], [1, 5])), 17
    if name == "hubs12":                    # degree 12: band bodies
        return bp.hubs(6, 12, ring=60), 0
    if name == "hubs13":                    # degree 13: 6 border bodies, 18 rows
        return bp.hubs(6, 13, ring=60), 18
    if name == "hubs12_obst":               # 12 two-body contacts + 3 one-body contacts each: still band bodies
        return bp.hubs(6, 12, ring=60, obstacle_per_hub=3), 0
    if name == "hub_links":                 # border-border contacts (the corner's atomics)
        return bp.hubs(5, 13, ring=60, hub_links=((0, 1), (1, 2), (4, 3), (0, 4), (2, 3))), 15
    if name == "hub40":
        return bp.hubs(1, 40, ring=61), 3
    if name == "hub300":
        return bp.hubs(1, 300, ring=301), 3
    if name in ("nband0", "nband1"):        # 4 bodies pinned by one row each: 4 x 3 + 4 = 16
        nb = 4 if name == "nband0" else 5
        pos = np.array([[0.0, 0.0], [2.0, 0.0], [0.0, 2.0], [2.0, 2.0], [4.0, 1.0]])[:nb]
        pairs = [(0, 1), (0, 2), (1, 3), (2, 3), (0, 3)] + ([(1, 4), (4, 3)] if nb == 5 else [])
        sc = bp.contacts_from_positions(pos, pairs, obstacle_pairs=[(2, 0.01)])
        return _with_rows(sc, _pin_rows(nb, [0, 4, 8, 10])), 16
    raise KeyError(name)


@pytest.mark.parametrize("name", ["border16", "border17", "hubs12", "hubs13", "hubs12_obst", "hub_links", "hub40",
                                  "hub300", "nband0", "nband1"])
def test_border(forced_banded, name):
    sc, nbd = _border_scene(name)
    o = bp.order_scene(sc)
    assert o["nbd"] == nbd, (o["nbd"], o["nbb"])
    if name == "nband0":
        assert o["nband"] == 0
    if name == "nband1":
        assert o["nband"] == 1
    if sc["nb"] * 3 + (sc["A"].shape[0] if "A" in sc else 0) <= 128:
        forced_banded(True)
    t = scene_inputs(sc, seed=11)
    if nbd > 16:
        assert kernel_bw(t, 1) == 0
        k = solve(t, 1, gz=torch.ones(t["v"].shape, dtype=f64))
        assert int(k["status"][0]) == -100
        assert all(float(g.abs().max()) == 0.0 for g in k["grads"].values())
        return
    check_oracle(t, 1, o)
    if sc["nb"] <= 70:
        check_oracle(t, 0, o, exacts=(False, True))


# ------------------------------------------------------------------------------------------ topology
def _components_scene():
    a = bp.lattice(5, 3, bp.FIVE)
    pos = np.concatenate([a["pos"], a["pos"] + 100.0, np.array([[500.0, 0.0], [600.0, 0.0], [700.0, 0.0]])])
    pairs = [(int(i), int(j)) for i, j in zip(a["body1"], a["body2"])]
    pairs += [(i + 15, j + 15) for i, j in pairs]
    return bp.contacts_from_positions(pos, pairs, obstacle_pairs=[(31, 0.01), (32, 0.02), (3, 0.01), (31, 0.03)])


@pytest.mark.parametrize("mode", [0, 1])
def test_components_isolated_and_obstacle_only_bodies(forced_banded, mode):
    sc = _components_scene()                     # two components, body 30 isolated, 31 / 32 touch only obstacles
    o = bp.order_scene(sc)
    assert o["nband"] == 33
    forced_banded(True)
    check_oracle(scene_inputs(sc, seed=13), mode, o, exacts=(False, True) if mode == 0 else (False,))


@pytest.mark.parametrize("nb", list(range(43, 51)))
def test_every_residue_of_nb(nb):
    """Nb = 3 nband over 8 consecutive body counts: every residue mod 8 (the identity padding of the last pass)."""
    sc = bp.random_graph(nb, 100 + nb, mean_deg=4.0)
    o = bp.order_scene(sc)
    assert o["nband"] == nb
    check_oracle(scene_inputs(sc, seed=nb), 1, o)


def test_zero_contact_scene_inside_banded_batch():
    sc = bp.random_graph(50, 3, mean_deg=8.0)
    nc = len(sc["body1"])
    t = scene_inputs(sc, B=3, seed=17)
    k3 = solve(t, 0, counts=[nc, 0, nc - 5])
    assert k3["status"].tolist()[1] == 2 and int(k3["iters"][1]) == 0
    Md = torch.stack([t["inertia"][1], t["mass"][1], t["mass"][1]], -1).reshape(-1)
    free = -(Md * t["v"][1] + DT * t["fext"][1]) / Md           # M z = -p (engines.py:35-49)
    assert rel(k3["z"][1], free) < 1e-12
    keep = [0, 2]
    t2 = {kk: (v[keep].contiguous() if torch.is_tensor(v) and v.dim() > 1 else v) for kk, v in t.items()}
    k2 = solve(t2, 0, counts=[nc, nc - 5])
    assert torch.equal(k2["z"], k3["z"][keep])


def test_pairs_with_two_contacts_are_reproducible(forced_banded):
    """Every horizontal neighbour pair of a lattice touches twice (two contact points): reproducible bitwise across
    calls, and equal to the oracle."""
    base = bp.lattice(12, 5, bp.FIVE)
    pos = base["pos"]
    pairs = [(int(i), int(j)) for i, j in zip(base["body1"], base["body2"])]
    sc = bp.contacts_from_positions(pos, pairs)
    # a second contact per horizontal pair, its points moved off the centre line
    extra = bp.contacts_from_positions(pos, [p for p in pairs if int(p[1]) == int(p[0]) + 1])
    for key in ("body1", "body2", "normal"):
        sc[key] = np.concatenate([sc[key], extra[key]])
    off = np.stack([-extra["normal"][:, 1], extra["normal"][:, 0]], 1) * 0.3
    sc["p1"] = np.concatenate([sc["p1"], extra["p1"] + off])
    sc["p2"] = np.concatenate([sc["p2"], extra["p2"] + off])
    o = bp.order_scene(sc)
    t = scene_inputs(sc, seed=19)
    gz = torch.randn(t["v"].shape, generator=torch.Generator().manual_seed(6), dtype=f64)
    forced_banded(True)                                        # n = 180 > 128 already; forced for clarity
    a, b = solve(t, 0, gz=gz), solve(t, 0, gz=gz)
    assert torch.equal(a["z"], b["z"])
    for name in NAMES:
        assert torch.equal(a["grads"][name], b["grads"][name]), name
    check_oracle(t, 0, o, exacts=(False, True))


def test_dense_reference_matches_assemble_dense():
    """The assembly above against scenes.assemble_dense on two-body scenes (mode 0)."""
    from lcp_physics_b200.scenes import assemble_dense, make_contact_soa
    soa = make_contact_soa(3, 12, 20, seed=4)
    ref = assemble_dense(soa, fd=2, e=0, dt=DT, gravity=10.0)
    t = dict(soa)
    t["fext"] = torch.zeros(3, 36, dtype=f64)
    t["fext"][:, 2::3] = 10.0 * soa["mass"]
    got = dense_lcp(t, 0)
    for name, a, r in zip("QpGh", got[:4], ref[:4]):
        assert torch.allclose(a, r, rtol=0, atol=1e-13), name
    assert torch.equal(got[6], ref[6])
