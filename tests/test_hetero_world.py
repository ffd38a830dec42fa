"""CPU: the host side of heterogeneous batches in `BatchedWorld` (per-scene active bodies and no-contact pairs).

* validation of the activity mask, of constraints with active and inactive bodies in one scene, and of per-scene
  no_contact lists (`check_active`, `check_constraint_activity`, `no_contact_masks`, `pack_bits`);
* a host restatement of the active walk's pair decode (csrc/lcp_contacts.cuh, find_contacts_kernel with ACTIVE):
  compaction of the scene's active bodies, then the closed form + fix-up over the compacted counts, thread by thread
  and chunk by chunk, equals the lexicographic pair list of the full body list filtered to active pairs.
"""
import math

import numpy as np
import pytest
import torch

from lcp_physics_b200.world import (FixedJoint, Joint, MAX_ACTIVE_BODIES, XConstraint, check_active,
                                    check_constraint_activity, mask_bits, no_contact_masks, pack_bits)

NT, ITEMS = 256, 4                       # lcp_contacts.cuh: threads per CTA, consecutive pairs per thread and chunk


def pairs_before(i, n):
    return i * (2 * n - i - 1) // 2


def active_walk_pairs(act, nd):
    """The pairs the ACTIVE walk visits for one scene, in visiting order, as the kernel computes them: act [nt] bool
    (dynamic bodies 0..nd-1, then obstacles)."""
    lst = [k for k in range(len(act)) if act[k]]           # the compacted list: active bodies in index order
    nd_s, nt_s = sum(1 for k in lst if k < nd), len(lst)
    npairs = pairs_before(nd_s, nt_s)
    imax = min(nd_s - 1, nt_s - 2)
    out = []
    for q0 in range(0, npairs, NT * ITEMS):
        for tid in range(NT):
            q = q0 + tid * ITEMS
            i = j = 0
            if q < npairs:
                t = 2.0 * nt_s - 1.0
                ii = int(math.floor((t - math.sqrt(t * t - 8.0 * q)) * 0.5))
                ii = min(max(ii, 0), imax)
                while ii + 1 <= imax and pairs_before(ii + 1, nt_s) <= q:
                    ii += 1
                while ii > 0 and pairs_before(ii, nt_s) > q:
                    ii -= 1
                i, j = ii, q - pairs_before(ii, nt_s) + ii + 1
            for u in range(ITEMS):
                if q + u < npairs:
                    out.append((lst[i], lst[j]))
                    j += 1
                    if j == nt_s:
                        i += 1
                        j = i + 1
    return out


def filtered_pairs(act, nd):
    nt = len(act)
    return [(i, j) for i in range(nd) for j in range(i + 1, nt) if act[i] and act[j]]


@pytest.mark.parametrize("nd,no", [(1, 0), (2, 0), (5, 3), (40, 0), (60, 6), (75, 4), (130, 0)])
def test_active_pair_decode_equals_filtered_lexicographic_pairs(nd, no):
    """random masks at several densities, including 0 and 1 active body; (75, 4) and (130, 0) span several 1024-pair
    chunks when most bodies are active"""
    g = np.random.default_rng(nd * 100 + no)
    nt = nd + no
    masks = [np.zeros(nt, bool), np.ones(nt, bool)]
    one = np.zeros(nt, bool)
    one[g.integers(nt)] = True
    masks.append(one)
    masks += [g.random(nt) < p for p in (0.1, 0.25, 0.5, 0.75, 0.95)]
    if no:
        only_obst = np.zeros(nt, bool)
        only_obst[nd:] = True
        masks.append(only_obst)                                # obstacles never pair: no pair at all
    chunks = 0
    for act in masks:
        got = active_walk_pairs(act, nd)
        assert got == filtered_pairs(act, nd), act.nonzero()
        chunks = max(chunks, -(-len(got) // (NT * ITEMS)))
    if nt >= 75:
        assert chunks >= 2


def test_pack_bits_sets_bit_k_of_word_k_over_32():
    g = torch.Generator().manual_seed(1)
    m = torch.rand(5, 70, generator=g) < 0.5
    w = pack_bits(m)
    assert w.dtype == torch.int32 and tuple(w.shape) == (5, 3)
    u = w.numpy().view(np.uint32)
    for s in range(5):
        for k in range(70):
            assert bool((int(u[s, k // 32]) >> (k % 32)) & 1) == bool(m[s, k])
    assert int(u[0, 2]) >> 6 == 0                               # bits beyond nt stay clear


def test_check_active_shapes_and_dtype():
    a = check_active([True, False, True], 4, 3)
    assert tuple(a.shape) == (4, 3) and a.is_contiguous() and a[:, 1].sum() == 0
    full = torch.rand(4, 3) < 0.5
    assert torch.equal(check_active(full, 4, 3), full)
    assert torch.equal(check_active(torch.tensor([[True], [False], [True], [True]]), 4, 3)[:, 2],
                       torch.tensor([True, False, True, True]))
    with pytest.raises(ValueError, match="bool mask"):
        check_active(torch.ones(4, 3), 4, 3)
    with pytest.raises(ValueError, match=r"\[4, 3\]"):
        check_active(torch.ones(4, 2, dtype=torch.bool), 4, 3)
    with pytest.raises(ValueError, match=r"\[4, 3\]"):
        check_active(torch.ones(5, 3, dtype=torch.bool), 4, 3)
    assert MAX_ACTIVE_BODIES == 8192


def test_constraints_with_active_and_inactive_bodies_in_one_scene_raise():
    cons = [Joint(0, None, [0.0, 0.0]), Joint(1, 0, [0.0, 1.0]), FixedJoint(2, 3), XConstraint(4)]
    act = torch.ones(3, 6, dtype=torch.bool)
    act[1, :2] = False                                          # the first chain wholly inactive in scene 1: fine
    act[2, 4] = False                                           # a one-body constraint on an inactive body: fine
    check_constraint_activity(cons, act)
    act[2, 3] = False                                           # FixedJoint(2, 3) half active in scene 2
    with pytest.raises(ValueError, match=r"constraint 2 \(FixedJoint of bodies \(2, 3\)\).*scene 2"):
        check_constraint_activity(cons, act)
    act = torch.ones(3, 6, dtype=torch.bool)
    act[1, 0] = False
    with pytest.raises(ValueError, match=r"constraint 1 \(Joint.*scene 1"):
        check_constraint_activity(cons, act)


def test_no_contact_masks_shared_and_per_scene():
    nt = 7
    w = no_contact_masks([(0, 1), (5, 2)], 3, nt)
    assert w.dim() == 1 and w.dtype == torch.int32 and w.numel() == (nt * nt + 31) // 32
    ii, jj = torch.triu_indices(nt, nt, 1)
    ex = mask_bits(w, nt, ii, jj)
    assert {(int(a), int(b)) for a, b in zip(ii[ex], jj[ex])} == {(0, 1), (2, 5)}
    u = w.numpy().view(np.uint32)
    for a, b in ((0, 1), (2, 5)):
        bit = a * nt + b
        assert (int(u[bit >> 5]) >> (bit & 31)) & 1
    ws = no_contact_masks([[(0, 1)], [], [(6, 3), (1, 2)]], 3, nt)
    assert tuple(ws.shape) == (3, (nt * nt + 31) // 32)
    assert torch.equal(ws[0], no_contact_masks([(0, 1)], 3, nt)) and int(ws[1].abs().sum()) == 0
    exs = mask_bits(ws, nt, ii, jj)
    assert tuple(exs.shape) == (3, ii.numel()) and int(exs.sum()) == 3
    assert {(int(a), int(b)) for a, b in zip(ii[exs[2]], jj[exs[2]])} == {(3, 6), (1, 2)}
    big = no_contact_masks([(0, 1), (8190, 8191)], 1, 8192)                   # the largest world: words, no [nt, nt]
    assert big.numel() == 8192 * 8192 // 32
    got = mask_bits(big, 8192, torch.tensor([8190, 0, 5]), torch.tensor([8191, 1, 6]))
    assert got.tolist() == [True, True, False]
    assert no_contact_masks([], 3, nt).dim() == 1                             # an empty shared list
    with pytest.raises(ValueError, match="out of range.*of scene 2"):
        no_contact_masks([[(0, 1)], [], [(0, 7)]], 3, nt)
    with pytest.raises(ValueError, match="names one body twice"):
        no_contact_masks([[(0, 1)], [(4, 4)], []], 3, nt)
    with pytest.raises(ValueError, match="one pair list per scene"):
        no_contact_masks([[(0, 1)], []], 3, nt)
    with pytest.raises(ValueError, match="out of range"):
        no_contact_masks([(0, 9)], 3, nt)
