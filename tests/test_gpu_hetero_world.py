"""GPU: heterogeneous batches in `BatchedWorld` -- per-scene active bodies and no-contact pairs.

* the walk over each scene's active bodies (lcpb200_contacts_active): with every body active and one shared mask it
  equals lcpb200_contacts bitwise (counts, pairs, feat, geometry); with random per-scene activity and masks it equals
  the walk of each scene's standalone sub-world (polygon scenes) and find_contacts_torch (circles and obstacles),
  fp32 and fp64;
* a heterogeneous batch (circle piles in an obstacle bin, boxes, 4- and 7-link chains, random subsets active, per-scene
  no_contact) steps as B independent worlds: each scene against a homogeneous world of its active bodies alone over 40
  steps, with identical contact counts and dt-halving history, positions to 1e-10 relative and frozen bodies bitwise
  unmoved; the same for a banded scene of 150 balls with 30 inactive, and for a scene without an active body;
* rollout gradients w.r.t. the active bodies' masses, friction and initial velocities equal the standalone worlds'
  (both adjoints) to 2e-6 of their scale, frozen bodies' parameters get exactly zero, and linearize() of the active
  block equals the standalone's to 1e-10.
"""
import ctypes

import pytest
import torch

from tests.test_gpu_polygons import polygon_walk, random_scene

pytestmark = pytest.mark.gpu
f64 = torch.float64


# ---------------------------------------------------------------------------------------------------- the walk
def active_walk(scs, dtype, cap, active=None, mask=None, stride=0, plain=False):
    """lcpb200_contacts_active on scenes of equal shapes (random_scene dicts); active [B, nt] bool or None, mask: int32
    words ([W] with stride 0, or [B, W]) or None. plain: lcpb200_contacts with the shared mask instead."""
    from lcp_physics_b200 import _lib
    from lcp_physics_b200.world import pack_bits, polygon_centroid
    lib = _lib.load()
    B = len(scs)
    st = lambda k: torch.stack([s[k] for s in scs]).to("cuda", dtype).contiguous()
    pos, rad, pv, ov = st("pos"), st("rad"), st("polys"), st("obst")
    nb, npoly, no = pos.shape[1], pv.shape[1], ov.shape[1]
    cen = lambda k: polygon_centroid(torch.stack([s[k] for s in scs]).to("cuda", f64)).to(dtype).contiguous()
    pcen, oref = cen("polys"), cen("obst")
    fr, rs = torch.full((B, nb), 0.5, dtype=dtype, device="cuda"), torch.zeros(B, nb, dtype=dtype, device="cuda")
    pfr, ofr = st("pfric"), st("ofric")
    prs, ors = torch.zeros_like(pfr), torch.zeros_like(ofr)
    i32 = lambda *s: torch.empty(*s, dtype=torch.int32, device="cuda")
    b1, b2, feat, counts = i32(B, cap), i32(B, cap), i32(B, cap), i32(B)
    new = lambda *s: torch.empty(B, cap, *s, dtype=dtype, device="cuda")
    geo = [new(2), new(2), new(2), new(), new(), new()]
    aw = pack_bits(active.cpu()).cuda() if active is not None else None
    mk = mask.cuda() if mask is not None else None
    ins = [_lib.ptr(t) for t in (pos, rad, fr, rs, pv, pcen, pfr, prs, ov, oref, ofr, ors, b1, b2, counts, feat)]
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    if plain:
        _lib.check(lib.lcpb200_contacts(_lib.dtype_code(dtype), B, nb, npoly, no, 6, cap, 0.1, *ins,
                                        *[_lib.ptr(t) for t in geo], _lib.ptr(mk), stream))
    else:
        _lib.check(lib.lcpb200_contacts_active(_lib.dtype_code(dtype), B, nb, npoly, no, 6, cap, 0.1, *ins,
                                               *[_lib.ptr(t) for t in geo], _lib.ptr(mk), stride, _lib.ptr(aw), stream))
    torch.cuda.synchronize()
    return dict(b1=b1, b2=b2, feat=feat, counts=counts, geo=geo)


def mask_words(pairs, nt):
    from lcp_physics_b200.world import no_contact_masks
    return no_contact_masks(pairs, 1, nt)


def sub_scene(sc, act):
    """the scene holding only the active bodies of sc (random_scene dict), and the map sub index -> body index"""
    nb, npoly = sc["pos"].shape[0], sc["polys"].shape[0]
    a = torch.as_tensor(act)
    ka, kp, ko = a[:nb].nonzero()[:, 0], a[nb:nb + npoly].nonzero()[:, 0], a[nb + npoly:].nonzero()[:, 0]
    sub = dict(sc, pos=sc["pos"][ka], rad=sc["rad"][ka], polys=sc["polys"][kp], pfric=sc["pfric"][kp],
               obst=sc["obst"][ko], ofric=sc["ofric"][ko])
    return sub, torch.cat([ka, kp + nb, ko + nb + npoly])


@pytest.mark.parametrize("dtype", [f64, torch.float32])
@pytest.mark.parametrize("sizes", [(14, 0, 0, 60.0), (12, 0, 3, 80.0), (3, 8, 2, 60.0), (10, 36, 4, 140.0)])
def test_all_active_walk_equals_lcpb200_contacts(dtype, sizes):
    """every body active, no mask or one shared mask (stride 0): bitwise the outputs of lcpb200_contacts (the mask
    walk when a mask is given, else the polygon walk); the last size spans two 1024-pair chunks"""
    from tests.test_gpu_joints import mask_walk
    nc, npoly, no, spread = sizes
    scs = [random_scene(300 + s, nc, npoly, no, spread) for s in range(5)]
    nt = nc + npoly + no
    cap = 1024
    ones = torch.ones(5, nt, dtype=torch.bool)
    full = polygon_walk(scs, dtype, cap)
    assert int(full["counts"].sum()) > 0
    for act in (None, ones):
        got = active_walk(scs, dtype, cap, act)
        for k in ("counts", "b1", "b2", "feat"):
            assert torch.equal(got[k], full[k]), k
        for a, b in zip(got["geo"], full["geo"]):
            assert torch.equal(a, b)
    excl = [(0, 1), (1, nt - 1), (2, 3)]
    if dtype == f64:
        ref = mask_walk(scs, dtype, cap, excl)
        got = active_walk(scs, dtype, cap, ones, mask_words(excl, nt), 0)
        for k in ("counts", "b1", "b2", "feat"):
            assert torch.equal(got[k], ref[k]), k
        for a, b in zip(got["geo"], ref["geo"]):
            assert torch.equal(a, b)


@pytest.mark.parametrize("dtype", [f64, torch.float32])
@pytest.mark.parametrize("sizes", [(3, 8, 2, 60.0), (10, 36, 4, 140.0), (30, 0, 3, 100.0)])
def test_active_walk_equals_each_scenes_standalone_walk(dtype, sizes):
    """random per-scene activity (including scenes with 0 and 1 active body) and per-scene masks: each scene's
    contacts, feat and geometry are bitwise those of the walk of the world holding only its active bodies, with the
    sub-world's body indices mapped back"""
    nc, npoly, no, spread = sizes
    B = 8
    scs = [random_scene(500 + s, nc, npoly, no, spread) for s in range(B)]
    nt = nc + npoly + no
    g = torch.Generator().manual_seed(nt)
    act = torch.rand(B, nt, generator=g) < torch.linspace(0.2, 1.0, B).unsqueeze(1)
    act[0] = False
    act[1] = False
    act[1, 0] = True
    cap = 1024
    full = polygon_walk(scs, dtype, cap)
    excl = []
    for s in range(B):                             # per scene, about a third of its unmasked contact pairs
        n = int(full["counts"][s])
        pr = sorted({(int(a), int(b)) for a, b in zip(full["b1"][s, :n].tolist(), full["b2"][s, :n].tolist())})
        excl.append(pr[::3])
    words = torch.stack([mask_words(e, nt) for e in excl])
    got = active_walk(scs, dtype, cap, act, words, int(words.shape[1]))
    assert int(got["counts"][0]) == 0 and int(got["counts"][1]) == 0
    seen = 0
    for s in range(2, B):
        sub, idx = sub_scene(scs[s], act[s])
        inv = {int(k): q for q, k in enumerate(idx.tolist())}
        sub_excl = [(inv[a], inv[b]) for a, b in excl[s] if a in inv and b in inv]
        nsub = len(idx)
        if sub["pos"].shape[0] + sub["polys"].shape[0] == 0:
            assert int(got["counts"][s]) == 0
            continue
        ref = active_walk([sub], dtype, cap, mask=mask_words(sub_excl, nsub) if sub_excl else None, plain=True)
        n = int(ref["counts"][0])
        assert int(got["counts"][s]) == n, s
        m = idx.cuda()
        assert torch.equal(got["b1"][s, :n], m[ref["b1"][0, :n].long()].int()), s
        assert torch.equal(got["b2"][s, :n], m[ref["b2"][0, :n].long()].int()), s
        assert torch.equal(got["feat"][s, :n], ref["feat"][0, :n]), s
        for a, b in zip(got["geo"], ref["geo"]):
            assert torch.equal(a[s, :n], b[0, :n]), s
        seen += n
    assert seen > 0


@pytest.mark.parametrize("dtype", [f64, torch.float32])
@pytest.mark.parametrize("with_obstacles", [False, True])
def test_per_scene_world_matches_find_contacts_torch(dtype, with_obstacles):
    """circle worlds (2 chunks of pairs), random activity and per-scene no_contact: the active walk's lists equal
    find_contacts_torch's"""
    from lcp_physics_b200.world import BatchedWorld, rect_vertices
    g = torch.Generator().manual_seed(7)
    B, nb = 8, 48 if dtype == f64 else 40                      # fp32: a condensed-kernel world (3 nb <= 128)
    pos = (torch.rand(B, nb, 2, generator=g, dtype=f64) * 80.0).to(dtype)
    ob = dict(obstacles=torch.stack([rect_vertices([40.0, 85.0], [100.0, 10.0]),
                                     rect_vertices([40.0, -8.0], [100.0, 10.0], 0.1)])) if with_obstacles else {}
    nt = nb + (2 if with_obstacles else 0)
    act = torch.rand(B, nt, generator=g) < 0.7
    act[3] = True
    excl = [[(int(a), int(b)) for a, b in torch.randint(0, nb, (6, 2), generator=g).tolist() if a != b]
            for _ in range(B)]
    if with_obstacles:
        excl[2] += [(1, nb), (5, nb + 1)]
    w = BatchedWorld(pos, 4.0, no_contact=excl, active=act, strict_no_penetration=False, device="cuda",
                     contact_capacity=512 if dtype == f64 else 256, **ob)
    assert w.per_scene and w.nc_stride > 0
    counts, b1, b2 = w.find_contacts_torch()
    assert torch.equal(counts, w.counts) and int(counts.sum()) > 0
    for s in range(B):
        n = int(counts[s])
        assert torch.equal(b1[s, :n], w.c_b1[s, :n]) and torch.equal(b2[s, :n], w.c_b2[s, :n]), s
        a = act[s].cuda()
        assert bool(a[w.c_b1[s, :n].long()].all() and a[w.c_b2[s, :n].long()].all())
        pairs = set(zip(w.c_b1[s, :n].tolist(), w.c_b2[s, :n].tolist()))
        assert not any((min(p), max(p)) in pairs for p in excl[s])


def test_per_scene_no_contact_without_active():
    """per-scene no_contact lists alone (every body active): the walk equals find_contacts_torch, and every scene steps
    as the world of the same bodies with its own list shared"""
    from lcp_physics_b200.world import BatchedWorld, rect_vertices
    g = torch.Generator().manual_seed(17)
    B, nb = 6, 20
    k = torch.arange(nb, dtype=f64)
    pos = torch.stack([12.0 + 12.0 * (k % 7), 60.0 - 12.0 * (k // 7)], 1).expand(B, -1, -1).contiguous()
    pos = pos + 0.5 * torch.rand(B, nb, 2, generator=g, dtype=f64)
    vel = torch.zeros(B, nb, 3, dtype=f64)
    vel[..., 1] = 15.0 * (torch.rand(B, nb, generator=g, dtype=f64) - 0.5)
    obst = torch.stack([rect_vertices([45.0, 75.0], [120.0, 10.0]), rect_vertices([-5.0, 40.0], [10.0, 130.0]),
                        rect_vertices([95.0, 40.0], [10.0, 130.0])])
    nocon = [[(a, b) for a in range(nb) for b in range(a + 1, nb + 3)
              if float(torch.rand(1, generator=g)) < 0.1] for _ in range(B)]
    nocon[0] = []
    kw = dict(rad=5.0, vel=vel, mass=1.0, obstacles=obst, gravity=100.0)
    w = BatchedWorld(pos, device="cuda", no_contact=nocon, **kw)
    assert w.per_scene and w.active is None and w.active_words is None and w.nc_stride > 0
    alone = [BatchedWorld(pos[s:s + 1], device="cuda", no_contact=nocon[s] or None,
                          **dict(kw, vel=vel[s:s + 1])) for s in range(B)]
    hits = 0
    for step in range(25):
        counts, b1, b2 = w.find_contacts_torch()
        assert torch.equal(counts, w.counts), step
        for s in range(B):
            n = int(counts[s])
            assert torch.equal(b1[s, :n], w.c_b1[s, :n]) and torch.equal(b2[s, :n], w.c_b2[s, :n]), (step, s)
            assert int(alone[s].counts[0]) == n and torch.equal(alone[s].c_b1[0, :n], w.c_b1[s, :n]), (step, s)
            pairs = set(zip(w.c_b1[s, :n].tolist(), w.c_b2[s, :n].tolist()))
            assert not pairs & set(nocon[s])
        hits += int(counts.sum())
        w.step()
        for s in range(B):
            alone[s].step()
            assert float(w.t[s]) == float(alone[s].t[0]), (step, s)
    for s in range(B):
        assert float((w.p[s] - alone[s].p[0]).abs().max() / alone[s].p[0].abs().max()) < 1e-10, s
    assert hits > 0


def test_entry_point_errors():
    from lcp_physics_b200 import _lib
    from lcp_physics_b200.world import BatchedWorld
    lib = _lib.load()
    i32 = torch.zeros(4, dtype=torch.int32, device="cuda")
    pos, rad = torch.zeros(1, 2, 2, dtype=f64, device="cuda"), torch.ones(1, 2, dtype=f64, device="cuda")
    args = lambda nb, feat, stride: (_lib.F64, 1, nb, 0, 0, 0, 4, 0.1, _lib.ptr(pos), _lib.ptr(rad), *[None] * 10,
                                     _lib.ptr(i32), _lib.ptr(i32), _lib.ptr(i32), feat, *[None] * 6, None, stride,
                                     None, None)
    assert lib.lcpb200_contacts_active(*args(8193, _lib.ptr(i32), 0)) != 0
    assert b"8192" in lib.lcpb200_last_error_string()
    assert lib.lcpb200_contacts_active(*args(2, None, 0)) != 0
    assert lib.lcpb200_contacts_active(*args(2, _lib.ptr(i32), -1)) != 0
    assert lib.lcpb200_contacts_active(*args(2, _lib.ptr(i32), 0)) == 0
    with pytest.raises(ValueError, match="8192"):
        BatchedWorld(torch.arange(8193 * 2, dtype=f64).reshape(1, 8193, 2) * 10, 1.0, active=True, device="cuda")
    with pytest.raises(ValueError, match="bool mask"):
        BatchedWorld(torch.zeros(2, 2, 2, dtype=f64), 1.0, active=torch.ones(2, 3, dtype=torch.bool), device="cuda")


# ---------------------------------------------------------------------------------------------------- worlds
def hetero_spec(B, seed, dtype=f64):
    """The union world: 12 circles of a pile and 4 boxes above them in a bin of 3 obstacles, a 4-link and a 7-link
    chain (Rect links hung from a world point, link joints, neighbours excluded from contact). Scene kinds: a random
    subset of the circles (and sometimes of the boxes) with the bin, or one chain alone."""
    from lcp_physics_b200.world import Joint, rect_vertices
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.rand(*s, generator=g, dtype=f64)
    cx = torch.tensor([15.0 + 22.0 * (k % 4) for k in range(12)], dtype=f64)
    cy = torch.tensor([60.0 - 13.0 * (k // 4) for k in range(12)], dtype=f64)
    pos = torch.stack([cx.expand(B, 12) + 2.0 * (r(B, 12) - 0.5), cy.expand(B, 12) + 1.0 * r(B, 12)], 2)
    vel = torch.zeros(B, 12, 3, dtype=f64)
    vel[..., 1] = 20.0 * (r(B, 12) - 0.5)
    rad = 4.5 + r(B, 12)
    boxes = [rect_vertices([15.0 + 25.0 * k, 8.0], [16.0, 10.0], 0.05 * k) for k in range(4)]
    links, cons, nocon = [], [], []
    for base, (nl, ax) in zip((4, 8), ((4, 300.0), (7, 420.0))):
        for k in range(nl):
            links.append(rect_vertices([ax, 50.0 + 50.0 * k], [16.0, 50.0]))
        cons.append(Joint(12 + base, None, [ax, 30.0]))
        for k in range(1, nl):
            cons.append(Joint(12 + base + k, 12 + base + k - 1, [ax, 25.0 + 50.0 * k]))
            nocon.append((12 + base + k, 12 + base + k - 1))
    polys = torch.stack(boxes + links)                                # [15, 4, 2]
    npoly = polys.shape[0]
    pvel = torch.zeros(B, npoly, 3, dtype=f64)
    pvel[:, 4:, 1] = 30.0 * (r(B, 11) - 0.5)                           # the chains swing
    pvel[:, :4, 0] = 0.2 * (r(B, 4) - 0.5)
    obst = torch.stack([rect_vertices([50.0, 75.0], [120.0, 10.0]), rect_vertices([-5.0, 40.0], [10.0, 130.0]),
                        rect_vertices([105.0, 40.0], [10.0, 130.0])])
    nd, nt = 12 + npoly, 12 + npoly + 3
    act = torch.zeros(B, nt, dtype=torch.bool)
    per_scene = []
    for s in range(B):
        kind = s % 4
        if kind in (0, 1):                                            # a pile: 4..12 circles, boxes in kind 1
            act[s, :12] = r(12) < 0.4 + 0.6 * r(1)
            act[s, int(torch.randint(0, 12, (1,), generator=g))] = True
            if kind == 1:
                act[s, 12:16] = r(4) < 0.7
            act[s, nd:] = True
            p = [(a, b) for a in range(12) for b in range(a + 1, 12) if r(1) < 0.05]
            per_scene.append(p)
        else:                                                         # one chain alone
            lo, nl = (16, 4) if kind == 2 else (20, 7)
            act[s, lo:lo + nl] = True
            per_scene.append([pr for pr in nocon if lo <= pr[1] < lo + nl])
    vel[~act[:, :12]] = 0.0                                          # inactive bodies at rest
    pvel[~act[:, 12:nd]] = 0.0
    mass = 0.5 + r(B, 12)
    pmass = 0.5 + r(B, npoly)
    kw = dict(pos=pos.to(dtype), rad=rad, vel=vel, mass=mass, fric_coeff=0.3 + 0.6 * r(B, 12), polygons=polys,
              poly_vel=pvel, poly_mass=pmass, obstacles=obst, constraints=cons, gravity=100.0, contact_capacity=64)
    return kw, act, per_scene


def sub_world_kwargs(kw, act, nocon, s):
    """The homogeneous one-scene world of the active bodies of scene s: bodies, constraints and no_contact pairs
    remapped to the sub-world's indices"""
    from lcp_physics_b200.world import FixedJoint, Joint
    nb, npoly = kw["pos"].shape[1], kw["polygons"].shape[-3] if "polygons" in kw else 0
    a = act[s]
    ka, kp, ko = a[:nb].nonzero()[:, 0], a[nb:nb + npoly].nonzero()[:, 0], a[nb + npoly:].nonzero()[:, 0]
    idx = torch.cat([ka, kp + nb, ko + nb + npoly])
    inv = {int(k): q for q, k in enumerate(idx.tolist())}
    one = lambda t, k: t[s:s + 1][:, k] if isinstance(t, torch.Tensor) and t.dim() >= 2 else t
    out = dict(pos=one(kw["pos"], ka), rad=one(kw["rad"], ka), vel=one(kw["vel"], ka), mass=one(kw["mass"], ka),
               fric_coeff=one(kw["fric_coeff"], ka), gravity=kw["gravity"])
    for k in ("dt", "post_stab", "exact_adjoint", "strict_no_penetration"):
        if k in kw:
            out[k] = kw[k]
    if len(kp):
        pv = kw["polygons"]
        out.update(polygons=pv[kp] if pv.dim() == 3 else pv[s:s + 1, kp], poly_vel=one(kw["poly_vel"], kp),
                   poly_mass=one(kw["poly_mass"], kp))
    if len(ko):
        ov = kw["obstacles"]
        out.update(obstacles=ov[ko] if ov.dim() == 3 else ov[s:s + 1, ko])
    cons = []
    for c in kw.get("constraints", []):
        if all(bool(a[k]) for k in c.bodies()):
            if isinstance(c, Joint):
                cons.append(Joint(inv[c.i], None if c.j is None else inv[c.j], c.anchor))
            elif isinstance(c, FixedJoint):
                cons.append(FixedJoint(inv[c.i], inv[c.j]))
            else:
                cons.append(type(c)(inv[c.i]))
    if cons:
        out["constraints"] = cons
    nc = [(inv[x], inv[y]) for x, y in nocon[s] if x in inv and y in inv]
    if nc:
        out["no_contact"] = nc
    return out, idx


def dyn_index(idx, nd):
    return idx[idx < nd]


def run_pair(kw, act, nocon, steps, scenes=None):
    """the heterogeneous world and the standalone worlds of its scenes (those with an active dynamic body), stepped
    together; checks counts and t at every step, frozen bodies at the end; returns the worlds"""
    from lcp_physics_b200.world import BatchedWorld
    w = BatchedWorld(device="cuda", active=act, no_contact=nocon, **kw)
    nd = w.nd
    scenes = range(w.B) if scenes is None else scenes
    alone = {}
    for s in scenes:
        sk, idx = sub_world_kwargs(kw, act, nocon, s)
        if len(dyn_index(idx, nd)):
            alone[s] = (BatchedWorld(device="cuda", **sk), dyn_index(idx, nd).cuda())
    p0, v0 = w.p.clone(), w.v.clone()
    frozen = ~w.body_active[..., 0]
    for k in range(steps):
        w.step()
        for s, (a, idx) in alone.items():
            a.step()
            assert int(w.counts[s]) == int(a.counts[0]), (k, s, int(w.counts[s]), int(a.counts[0]))
            assert float(w.t[s]) == float(a.t[0]), (k, s)                  # the same dt-halving history
    assert torch.equal(w.p[frozen], p0[frozen])
    fd = frozen.unsqueeze(2).expand(-1, -1, 3).reshape(w.B, w.n)
    assert torch.equal(w.v[fd], v0[fd])
    return w, alone


def rel_err(w, alone):
    worst = 0.0
    for s, (a, idx) in alone.items():
        d = (w.p[s, idx] - a.p[0]).abs().max() / a.p[0].abs().max().clamp_min(1.0)
        worst = max(worst, float(d))
    return worst


def test_heterogeneous_batch_equals_independent_worlds():
    kw, act, nocon = hetero_spec(64, 3)
    w, alone = run_pair(kw, act, nocon, 40)
    assert len(alone) == 64
    err = rel_err(w, alone)
    print("heterogeneous batch of 64 vs standalone worlds, 40 steps: max rel position error %.2e, contacts %d"
          % (err, int(w.counts.sum())))
    assert err < 1e-10
    assert not w.large


def test_heterogeneous_batch_with_post_stabilisation():
    kw, act, nocon = hetero_spec(8, 5)
    kw["post_stab"] = True
    w, alone = run_pair(kw, act, nocon, 15)
    assert rel_err(w, alone) < 1e-10


def test_large_banded_scene_with_inactive_balls_equals_its_sub_world():
    from lcp_physics_b200.world import rect_vertices
    g = torch.Generator().manual_seed(9)
    nb, cols = 150, 15
    k = torch.arange(nb, dtype=f64)
    pos = torch.stack([10.0 + 11.0 * (k % cols) + 0.5 * torch.rand(nb, generator=g, dtype=f64),
                       200.0 - 11.0 * (k // cols)], 1).unsqueeze(0).expand(2, -1, -1).contiguous()
    obst = torch.stack([rect_vertices([87.0, 211.0], [200.0, 10.0]), rect_vertices([-2.0, 120.0], [8.0, 200.0]),
                        rect_vertices([176.0, 120.0], [8.0, 200.0])])
    act = torch.ones(2, nb + 3, dtype=torch.bool)
    act[0, torch.randperm(nb, generator=g)[:30]] = False
    full = lambda v: torch.full((2, nb), v, dtype=f64)
    kw = dict(pos=pos, rad=full(5.0), vel=torch.zeros(2, nb, 3, dtype=f64), mass=full(1.0), fric_coeff=full(0.9),
              obstacles=obst, gravity=100.0)
    w, alone = run_pair(kw, act, [[], []], 12)
    assert w.large and alone[0][0].large
    err = rel_err(w, alone)
    print("150-ball banded scene with 30 inactive vs its 120-ball sub-world: max rel position error %.2e" % err)
    assert err < 1e-10


def test_scene_without_active_body():
    kw, act, nocon = hetero_spec(4, 8)
    act[1] = False
    act[2] = False
    act[2, 0] = True                                                  # one ball alone
    kw["vel"][1] = 5.0                                                # frozen with a velocity: carried unchanged
    w, alone = run_pair(kw, act, nocon, 6)
    assert int(w.counts[1]) == 0 and abs(float(w.t[1]) - 6 * w.dt) < 1e-15
    assert rel_err(w, alone) < 1e-10


def test_inactive_joint_keeps_its_state():
    """a wholly inactive chain whose links carry a velocity: the bodies and their joints' state stay as they were"""
    kw, act, nocon = hetero_spec(4, 12)
    pv = kw["poly_vel"].clone()
    pv[0, 4:] = torch.tensor([0.5, 3.0, -2.0], dtype=f64)           # scene 0 is a pile: both chains inactive, moving
    kw["poly_vel"] = pv
    from lcp_physics_b200.world import BatchedWorld
    w = BatchedWorld(device="cuda", active=act, no_contact=nocon, **kw)
    before = [None if st is None else [t.clone() for t in st[1:]] for st in w._jstate]
    p0 = w.p.clone()
    for _ in range(5):
        w.step()
    assert torch.equal(w.p[0, 16:], p0[0, 16:]) and torch.equal(w.v[0, 48:], pv[0, 4:].reshape(-1).cuda())
    for st, old in zip(w._jstate, before):
        for t, o in zip(st[1:], old):
            assert torch.equal(t[0], o[0])
    moved = [not torch.equal(st[1][2], old[0][2]) for st, old in zip(w._jstate, before)]
    assert any(moved)                                                  # scene 2 swings its 4-link chain


def test_active_none_and_all_active_equal_todays_world():
    """active=None takes today's path (lcpb200_contacts); an all-true mask the active walk, with the same steps"""
    from lcp_physics_b200.world import BatchedWorld
    kw, act, nocon = hetero_spec(8, 4)
    kw.pop("constraints")
    kw["polygons"] = kw["polygons"][:4]
    kw["poly_vel"], kw["poly_mass"] = kw["poly_vel"][:, :4], kw["poly_mass"][:, :4]
    w0 = BatchedWorld(device="cuda", **kw)
    w1 = BatchedWorld(device="cuda", active=None, **kw)
    w2 = BatchedWorld(device="cuda", active=True, **kw)
    assert not w1.per_scene and w1.active is None and w2.per_scene
    for _ in range(10):
        for w in (w0, w1, w2):
            w.step()
        assert torch.equal(w0.counts, w1.counts) and torch.equal(w0.counts, w2.counts)
        assert torch.equal(w0.p, w1.p) and torch.equal(w0.c_b1, w2.c_b1)
        assert float((w0.p - w2.p).abs().max()) < 1e-9


# ---------------------------------------------------------------------------------------------------- gradients
def pile_spec(B, seed):
    kw, act, nocon = hetero_spec(B, seed)
    for k in ("constraints", "polygons", "poly_vel", "poly_mass"):
        kw.pop(k)
    act = torch.cat([act[:, :12], act[:, -3:]], 1)
    for s in range(B):
        if not act[s, :12].any():
            act[s, :6] = True
        act[s, 12:] = True
    kw["pos"] = kw["pos"] + torch.tensor([0.0, 3.0], dtype=kw["pos"].dtype)   # the bottom row 0.5-2 above the floor
    kw["vel"] = kw["vel"].clone()
    kw["vel"][..., 1] = 8.0 * act[:, :12] * (1 - 2 * (torch.arange(12) % 2))      # sliding on the floor
    return kw, act, [[] for _ in range(B)]


def box_spec(B, seed):
    """4 boxes sliding on the bin's floor, random subsets active: friction decides their motion"""
    from lcp_physics_b200.world import rect_vertices
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.rand(*s, generator=g, dtype=f64)
    boxes = torch.stack([rect_vertices([15.0 + 25.0 * k, 64.9], [16.0, 10.0]) for k in range(4)])
    act = torch.ones(B, 7, dtype=torch.bool)
    act[:, :4] = r(B, 4) < 0.6
    act[:, 0] |= ~act[:, :4].any(1)
    pvel = torch.zeros(B, 4, 3, dtype=f64)
    pvel[..., 1] = 20.0 * (1 - 2 * (torch.arange(4) % 2)) * (0.5 + r(B, 4)) * act[:, :4]
    obst = torch.stack([rect_vertices([50.0, 75.0], [120.0, 10.0]), rect_vertices([-5.0, 40.0], [10.0, 130.0]),
                        rect_vertices([105.0, 40.0], [10.0, 130.0])])
    kw = dict(pos=torch.zeros(B, 0, 2, dtype=f64), rad=torch.zeros(B, 0, dtype=f64),
              polygons=boxes.expand(B, -1, -1, -1).contiguous(), poly_vel=pvel, poly_mass=0.5 + r(B, 4),
              poly_fric=0.2 + 0.6 * r(B, 4), obstacles=obst, gravity=100.0)
    return kw, act


def parked(kw, act, leaves):
    """The same batch without `active`: every inactive body parked far from everything (a distinct spot per body),
    at rest, its gravity cancelled by an external force, so that the dof layout is that of the heterogeneous world"""
    from lcp_physics_b200.world import BatchedWorld
    B, nb = kw["pos"].shape[:2]
    npoly = kw["polygons"].shape[1] if "polygons" in kw else 0
    off = ~act[:, :nb + npoly]
    spot = lambda k: torch.tensor([1.0e4 + 200.0 * k, 1.0e4], dtype=f64)
    pos = kw["pos"].clone()
    for s, k in off[:, :nb].nonzero().tolist():
        pos[s, k] = spot(k)
    extra = {}
    if npoly:
        pv = kw["polygons"].clone()
        for s, k in off[:, nb:].nonzero().tolist():
            pv[s, k] = pv[s, k] - pv[s, k].mean(0) + spot(nb + k)
        extra["polygons"] = pv
    args = dict(kw, pos=pos, **extra, **leaves)
    w = BatchedWorld(device="cuda", **args)
    cancel = torch.zeros(B, nb + npoly, 3, dtype=f64, device="cuda")
    cancel[..., 2] = -w.fext[:, 2::3] * off.cuda()                  # m g - m g = 0 exactly
    w.external_force = lambda t: cancel
    return w


def rollout_grads(w, wt, names, leaves, steps):
    for _ in range(steps):
        w.step()
    nd = wt.shape[1]
    return w, torch.autograd.grad((w.p[:, :nd] * wt).sum(), [leaves[k] for k in names])


@pytest.mark.parametrize("exact", [False, True])
@pytest.mark.parametrize("kind", ["piles", "boxes"])
def test_rollout_gradients_equal_the_parked_layout(kind, exact):
    """rollout gradients w.r.t. the active bodies' masses, friction and initial velocities equal (1e-9) those of the
    same batch with the inactive bodies parked instead of frozen -- the same dof layout -- and frozen bodies'
    parameters get exactly zero. Boxes slide on the floor: friction decides their motion."""
    from lcp_physics_b200.world import BatchedWorld
    if kind == "piles":
        kw, act, _ = pile_spec(6, 21)
        names, nd, steps = ("mass", "fric_coeff", "vel"), 12, 20
    else:
        kw, act = box_spec(6, 5)
        names, nd, steps = ("poly_mass", "poly_fric", "poly_vel"), 4, 15
    kw["exact_adjoint"] = exact
    B = act.shape[0]
    wt = torch.randn(B, nd, 3, generator=torch.Generator().manual_seed(0), dtype=f64).cuda()
    wt = wt * act[:, :nd].cuda()[..., None]
    lh = {k: kw[k].clone().requires_grad_(True) for k in names}
    wh, gh = rollout_grads(BatchedWorld(device="cuda", active=act, **dict(kw, **lh)), wt, names, lh, steps)
    lp = {k: kw[k].clone().requires_grad_(True) for k in names}
    wp, gp = rollout_grads(parked(kw, act, lp), wt, names, lp, steps)
    on = act[:, :nd]
    assert torch.equal(wh.counts, wp.counts) and torch.equal(wh.t, wp.t)
    # the parameters that decide the motion: piles fall and roll (mass, velocity), boxes slide (friction, velocity;
    # a sliding box's motion does not depend on its mass)
    deciding = (0, 2) if kind == "piles" else (1, 2)
    scales = [float(b[on].abs().max()) for b in gp]
    assert all(scales[q] > 1e-3 for q in deciding), scales
    errs = []
    for q, (a, b) in enumerate(zip(gh, gp)):
        assert bool((a[~on] == 0).all()), names[q]
        errs.append(float((a[on] - b[on]).abs().max()) / max(scales[q], 1e-3 * max(scales)))
    print("%s, exact_adjoint=%s: rollout gradients vs the parked layout, max |diff| / scale %s"
          % (kind, exact, ["%.1e" % e for e in errs]))
    assert max(errs) < 1e-9


@pytest.mark.parametrize("exact", [False, True])
def test_rollout_gradients_equal_standalone_worlds(exact):
    """the same pile rollouts against each scene's standalone world of its active bodies. A smaller KKT system
    changes the order of the round-off in the solves; these solves stop at the PDIPM tolerance, whose adjoint
    amplifies it. The test measures that amplification with no `active` involved -- the standalone world against
    itself with one isolated, gravity-free ball inserted in front of its bodies -- and gates the heterogeneous world
    at 2e-6 of the gradient scale, above both."""
    from lcp_physics_b200.world import BatchedWorld
    B, steps = 6, 20
    kw, act, nocon = pile_spec(B, 21)
    kw["exact_adjoint"] = exact
    names = ("mass", "fric_coeff", "vel")
    leaves = {k: kw[k].clone().requires_grad_(True) for k in names}
    wt = torch.randn(B, 12, 3, generator=torch.Generator().manual_seed(0), dtype=f64).cuda()
    w, grads = rollout_grads(BatchedWorld(device="cuda", active=act, **dict(kw, **leaves)),
                             wt * act[:, :12].cuda()[..., None], names, leaves, steps)
    diff, ref, scale = [0.0] * 3, [0.0] * 3, [0.0] * 3
    for s in range(B):
        sk, idx = sub_world_kwargs(kw, act, nocon, s)
        ka = idx[idx < 12]
        ws = wt[s:s + 1, ka.cuda()]
        sl = {k: sk[k].clone().requires_grad_(True) for k in names}
        _, ga = rollout_grads(BatchedWorld(device="cuda", **dict(sk, **sl)), ws, names, sl, steps)
        # the standalone world with one isolated, gravity-free ball in front of its bodies
        k = len(ka)
        front = lambda t, v: torch.cat([torch.full_like(t[:, :1], v), t], 1)
        si = dict(sk, pos=torch.cat([torch.tensor([[[5000.0, 5000.0]]], dtype=f64), sk["pos"]], 1),
                  rad=front(sk["rad"], 5.0), gravity_mask=[False] + [True] * k)
        li = dict(mass=front(sk["mass"], 1.0), fric_coeff=front(sk["fric_coeff"], 0.5),
                  vel=torch.cat([torch.zeros(1, 1, 3, dtype=f64), sk["vel"]], 1))
        li = {q: v.requires_grad_(True) for q, v in li.items()}
        _, gi = rollout_grads(BatchedWorld(device="cuda", **dict(si, **li)),
                              torch.cat([torch.zeros_like(ws[:, :1]), ws], 1), names, li, steps)
        for q in range(3):
            diff[q] = max(diff[q], float((grads[q][s:s + 1][:, ka] - ga[q]).abs().max()))
            ref[q] = max(ref[q], float((gi[q][:, 1:] - ga[q]).abs().max()))
            scale[q] = max(scale[q], float(ga[q].abs().max()))
        for g_full in grads:
            assert bool((g_full[s][~act[s, :12]] == 0).all()), s
    # mass and velocity: relative to their scale; friction gradients of these rolling piles are at round-off level
    # (boxes sliding test friction against the parked layout), so they are bounded relative to the mass scale
    err = lambda d: [d[0] / scale[0], d[1] / scale[0], d[2] / scale[2]]
    print("piles, exact_adjoint=%s: rollout gradients vs standalone (mass, friction, velocity) %s; standalone with an "
          "isolated ball in front vs standalone %s; scales %s" % (exact, ["%.1e" % e for e in err(diff)],
                                                                 ["%.1e" % e for e in err(ref)],
                                                                 ["%.3g" % v for v in scale]))
    assert scale[0] > 1e-3 and scale[2] > 1e-3 and max(err(diff)) < 2e-6


def test_linearize_active_block_equals_standalone():
    from lcp_physics_b200.world import BatchedWorld
    B = 4
    kw, act, nocon = pile_spec(B, 22)
    kw["exact_adjoint"] = True
    w = BatchedWorld(device="cuda", active=act, **kw)
    for _ in range(3):
        w.step()
    x1, A, Bu = w.linearize()
    n = w.n
    for s in range(B):
        sk, idx = sub_world_kwargs(kw, act, nocon, s)
        a = BatchedWorld(device="cuda", **sk)
        for _ in range(3):
            a.step()
        xa, Aa, Ba = a.linearize()
        kd = idx[idx < 12]
        dofs = (3 * kd.unsqueeze(1) + torch.arange(3)).reshape(-1).cuda()
        rows = torch.cat([dofs, dofs + n])
        blk = A[s][rows][:, rows]
        err = float((blk - Aa[0]).abs().max() / Aa[0].abs().max())
        assert err < 1e-10, (s, err)
        assert float((Bu[s][rows][:, dofs] - Ba[0]).abs().max() / Ba[0].abs().max()) < 1e-10
        off = torch.ones(2 * n, dtype=torch.bool, device="cuda")
        off[rows] = False
        eye = torch.eye(2 * n, dtype=f64, device="cuda")
        assert torch.equal(A[s][off], eye[off]) and bool((Bu[s][off] == 0).all())
