"""Shared test helpers: golden fixture loading, error metrics, the fp32 accuracy gate and the dual-form switch."""
import contextlib
import glob
import os

import numpy as np
import torch


@contextlib.contextmanager
def dual_only():
    """Plan new handles without the condensed-KKT kernels (the dense / dual-form path)."""
    from lcp_physics_b200 import _lib
    os.environ["LCPB200_NO_CONDENSED"] = "1"
    _lib.clear_handles()
    try:
        yield
    finally:
        del os.environ["LCPB200_NO_CONDENSED"]
        _lib.clear_handles()


def fp32_gate(zhat, ref32, ref64, what):
    """Distributional fp32 accuracy gate (tests/test_gpu_parity.py's module docstring): zhat against the fp32 and
    the fp64 reference of the same scenes."""
    err = rel_err(zhat, ref32)
    own = rel_err(ref32, ref64)
    mine = rel_err(zhat, ref64)
    assert float((err <= 1e-3 + 1.5 * own).float().mean()) >= 0.95, (what, err, own)
    assert float((err < 1e-3).float().mean()) >= 0.85, (what, err)
    assert float(err.max()) <= 2e-2, (what, err)
    assert float(mine.median()) <= 1.2 * float(own.median()) + 1e-6, (what, mine.median(), own.median())
    assert float(mine.quantile(0.9)) <= 1.2 * float(own.quantile(0.9)) + 1e-4, (what, mine.quantile(0.9), own.quantile(0.9))

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def golden_names():
    return sorted(n for n in (os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN_DIR, "*.npz")))
                  if not n.startswith(("world_", "seeded_", "bworld_")))


def seeded_names():
    return sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN_DIR, "seeded_*.npz")))


def load_seeded_golden(name):
    """Fixtures of tests/golden/make_seeded_golden.py: outputs of the unmodified reference on 48 seeded scenes
    at a BASELINE shape, with the inputs stored in packed form (non-zero pattern once, values per scene).
    Returns (fp64 inputs, {"f64": outputs, "f32": outputs}, max_iter, dl_dzhat)."""
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    B = int(z["kwargs"][0])
    inp = []
    for k in "Q p G h A b F".split():
        if "in_" + k + "_idx" in z.files:
            shape = tuple(int(v) for v in z["in_" + k + "_shape"])
            flat = torch.zeros(B, int(np.prod(shape)), dtype=torch.float64)
            flat[:, torch.from_numpy(z["in_" + k + "_idx"].astype(np.int64))] = torch.from_numpy(z["in_" + k + "_val"])
            inp.append(flat.reshape((B,) + shape))
        else:
            inp.append(torch.tensor([], dtype=torch.float64))          # e == 0: 1-D empty A, b (engines.py:59-60)
    out = {tag: {k[len(tag) + 1:]: torch.from_numpy(z[k]) for k in z.files if k.startswith(tag + "_")}
           for tag in ("f64", "f32")}
    return tuple(inp), out, int(z["max_iter"]), torch.from_numpy(z["dl_dzhat"])


def load_golden(name, dtype=torch.float64):
    """Returns (inputs tuple, dict of reference outputs for that dtype, max_iter, dl_dzhat)."""
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    inputs = tuple(torch.from_numpy(z["in_" + k]).to(dtype) for k in "Q p G h A b F".split())
    tag = "f64" if dtype == torch.float64 else "f32"
    out = {k[len(tag) + 1:]: torch.from_numpy(z[k]) for k in z.files if k.startswith(tag + "_")}
    return inputs, out, int(z["max_iter"]), torch.from_numpy(z["dl_dzhat"]).to(dtype)


def rel_err(a, b):
    """Per-scene relative 2-norm error, flattened over non-batch dims."""
    a = a.double().reshape(a.shape[0], -1)
    b = b.double().reshape(b.shape[0], -1)
    return (a - b).norm(dim=1) / b.norm(dim=1).clamp_min(1e-300)


class _ReplayBody:
    def __init__(self, fric, rest):
        self.fric_coeff = fric
        self.restitution = rest


class ReplayWorld:
    """Stand-in for the reference `World` holding exactly what an engine reads from it
    (engines.py:27-77), rebuilt from one record of tests/golden/world_*.npz."""

    def __init__(self, rec, dtype=torch.float64):
        t = lambda a: torch.from_numpy(np.asarray(a)).to(dtype)
        self.t = float(rec["t"])
        self._M, self._Je, self._v, self._f = t(rec["M"]), t(rec["Je"]), t(rec["v"]), t(rec["f"])
        self.vec_len = 3
        self.fric_dirs = 2
        self.static_inverse = True
        self.bodies = [_ReplayBody(float(f), float(r)) for f, r in zip(rec["fric"], rec["rest"])]
        nrm, p1, p2 = t(rec["normal"]), t(rec["p1"]), t(rec["p2"])
        self.contacts = [((nrm[i], p1[i], p2[i], torch.zeros(1, dtype=dtype)), int(rec["b1"][i]), int(rec["b2"][i]))
                         for i in range(len(rec["b1"]))]

    def M(self):
        return self._M

    def Je(self):
        return self._Je

    def get_v(self):
        return self._v

    def apply_forces(self, t):
        return self._f


def load_world_records(name):
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    out = []
    for i in range(int(z["count"])):
        pre = "%03d_" % i
        out.append({k[len(pre):]: z[k] for k in z.files if k.startswith(pre)})
    return out
