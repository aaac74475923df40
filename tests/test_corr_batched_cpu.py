"""f4, batched retrieval on the CPU: the HOST build of ``corr_retrieve_query`` (csrc/corr_core.cuh through
tests/host_harness/corr_retrieve_host.cpp, the arithmetic of ``bxs_corr_retrieve``) against a sequential replay of the oracle's
``Queues.similar`` / ``append`` over multi-level, multi-class sequences (tests/corr_sequences.py): every level is resolved in
one call, and object i must retrieve exactly the slots the oracle retrieves after the objects before it -- those of its own
level included -- were appended.  The GPU twin is tests/test_corr_batched_gpu.py."""
import ctypes

import pytest
import torch

from oracle.make_golden_corr import CH, FEAT, MASK
from tests import corr_sequences as cs
from tests.helpers import host_twin


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def host_retrieve(store, first, s_feat, s_feat_first, s_mask, t_feat, t_mask, boxes, labels, valid, min_objs=5):
    feat, mask, box, ptr, exists = store
    n, K = s_feat.shape[0], cs.BANK['max_retrieval_objs']
    src = torch.full((n, K), -7, dtype=torch.int32)
    count, kcount, slot, exq = [torch.full((n,), -7, dtype=torch.int32) for _ in range(4)]
    flag = torch.tensor([int(first)], dtype=torch.int32)
    lab, val = labels.to(torch.int32).contiguous(), valid.to(torch.int32).contiguous()
    args = [feat, mask, box, ptr, exists, flag, s_feat, s_feat_first, s_mask, t_feat, t_mask, boxes, lab, val, src, count, kcount,
            slot, exq]
    args = [a.contiguous() for a in args]
    lib = host_twin('corr_retrieve_host')
    b = cs.BANK
    rc = lib.host_corr_retrieve(*[_p(a) for a in args], *[ctypes.c_int64(v) for v in (n, cs.NUM_CLASS, b['len_queue'], CH, FEAT,
                                                                                         FEAT, MASK, MASK)],
                                *[ctypes.c_float(v) for v in (b['fg_iou_thresh'], b['bg_iou_thresh'], b['appear_thresh'],
                                                              b['ratio_range'][0], b['ratio_range'][1], cs.MIN_SIZE)],
                                ctypes.c_int(K), ctypes.c_int(min_objs))
    assert rc == 0
    return args[14], args[15], args[16], args[17], args[18]


def host_append(store, s_level, slot, labels, valid):
    """What bxs_corr_bank_append does, on the packed CPU store (the order of the level, last writer wins)."""
    feat, mask, box, ptr, exists = store
    _, t_feat, _, t_mask, boxes, _, _ = s_level
    L = cs.BANK['len_queue']
    for i in range(len(slot)):
        if slot[i] >= 0:
            c = int(labels[i])
            row = c * L + int(slot[i])
            feat[row], mask[row], box[row] = t_feat[i], t_mask[i], boxes[i]
            ptr[c], exists[c] = (int(slot[i]) + 1) % L, 1


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_host_retrieval_equals_sequential_oracle(seed):
    from oracle import corr as oc
    orc, levels = cs.sequence(seed)
    store = list(cs.packed(orc))
    first = True
    margin, passing, failing, in_level, retrieved, created = float('inf'), 0, 0, 0, 0, 0
    for lv in levels:
        s_feat, t_feat, s_mask, t_mask, boxes, labels, valid = lv
        had_bank = [orc.banks[int(c)] is not None for c in labels]
        src, count, kcount, slot, exq = host_retrieve(store, first, s_feat, oc.relu_and_l2_norm_feat(s_feat), s_mask, t_feat,
                                                      t_mask, boxes, labels, valid)
        want, appends, m, p, f, first_after = cs.replay(orc, first, *lv)
        margin, passing, failing = min(margin, m), passing + p, failing + f
        assert slot.tolist() == appends
        for i, w in enumerate(want):
            if w is None:
                assert int(count[i]) == 0 and int(kcount[i]) == 0
                assert int(exq[i]) == 0 or not bool(valid[i])
                continue
            assert int(exq[i]) == 1
            got = cs.decode(src[i], count[i], slot)
            assert got == w, (i, got, w)
            assert int(kcount[i]) == (len(w) if len(w) >= 5 else 0)
            in_level += sum(1 for s in src[i, :int(count[i])] if s < 0)
            retrieved += len(w)
        created += sum(1 for h, w in zip(had_bank, want) if not h and w is not None)   # class created earlier in the level
        host_append(store, lv, slot, labels, valid)
        first = first_after
        for c, b in enumerate(orc.banks):                                 # the store after the level == the oracle's bank
            L = cs.BANK['len_queue']
            if b is not None:
                assert torch.equal(store[0][c * L:(c + 1) * L], b.feature) and torch.equal(store[1][c * L:(c + 1) * L], b.mask)
                assert torch.equal(store[2][c * L:(c + 1) * L], b.box) and int(store[3][c]) == b.ptr and int(store[4][c]) == 1
            else:
                assert int(store[4][c]) == 0
    assert margin >= 1e-5, margin                                         # no decision within rounding of its threshold
    assert passing > 0 and failing > 0 and in_level > 0 and retrieved >= 10 and created > 0


def test_invalid_and_out_of_range_objects_take_no_part():
    orc, levels = cs.sequence(0)
    store = list(cs.packed(orc))
    s_feat, t_feat, s_mask, t_mask, boxes, labels, valid = levels[0]
    labels = labels.clone()
    labels[0] = cs.NUM_CLASS                                              # outside [0, num_class)
    valid = torch.zeros_like(valid)
    valid[0] = True
    src, count, kcount, slot, exq = host_retrieve(store, True, s_feat, s_feat, s_mask, t_feat, t_mask, boxes, labels, valid)
    assert (count == 0).all() and (kcount == 0).all() and (slot == -1).all() and (exq == 0).all() and (src == 0).all()
