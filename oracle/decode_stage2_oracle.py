"""ORACLE — test infrastructure only (never imported by the product path).

Numpy restatement of the SECOND stage of the reference's per-site decoder, the part ``c3b_decode_stage2``
(clair3_b200/csrc/decode.cu) runs on the GPU: the outcome lists ``possible_outcome_probabilites_from`` builds
(``clair3/CallVariants.py:413-494`` with the indel-length heads, ``:519-562`` without) and the order in which
``output_from`` (``:720-1005``) tries their entries.

``output_from`` repeatedly takes the maximum over all lists, returns a reference call if it equals ``homo_Ref_probability``,
otherwise tries the first index holding it in the first category (``elif`` order) that holds it, and zeroes that entry when
the alt-info check fails.  So the order of attempts depends on ``y`` only: probability descending, then category, then
index.  Categories are numbered in the ``elif`` order, homo_Ref first (``CATEGORIES``); within a category an entry's index is
its position in the reference's list (hetero_DelDel: list order, not the sorted length tuple).

Pinned by ``tests/golden/decode_stage2.npz``, minted by ``tests/golden/make_decode_stage2_golden.py`` from the reference's own
``output_from`` with its alt-info helpers replaced by recording stubs that always fail.
"""
from __future__ import annotations

import numpy as np

CATEGORIES = ("homo_Ref", "homo_SNP", "hetero_SNP", "homo_Ins", "hetero_ACGT_Ins", "hetero_InsIns", "homo_Del",
              "hetero_ACGT_Del", "hetero_DelDel", "hetero_InsDel")
CAT_SIZES = {90: (1, 4, 6, 16, 64, 136, 16, 64, 241, 256), 24: (1, 4, 6, 1, 4, 1, 1, 4, 1, 1)}
HOMO_SNP_GT21 = (0, 4, 7, 9)                     # AA CC GG TT                  clair3/task/gt21.py
HETERO_SNP_GT21 = (1, 2, 3, 5, 6, 8)             # AC AG AT CG CT GT
GT21_DELDEL, GT21_ADEL, GT21_INSINS, GT21_AINS, GT21_INSDEL = 10, 11, 15, 16, 20
INSINS_PAIRS = [(i, j) for i in range(1, 17) for j in range(i, 17)]                              # :320-330
DELDEL_PAIRS = [(i, j) for i in range(1, 17) for j in range(1, 17) if not (i == j and i != 16)]  # :349-360, list order
INSDEL_PAIRS = [(i, j) for i in range(1, 17) for j in range(1, 17)]                              # :363-372
PAD_CAT = 255


def category_of_slot(out_dim):
    """Slot s of the concatenated lists -> (category, index within the category's list)."""
    cat = np.repeat(np.arange(10, dtype=np.uint8), CAT_SIZES[out_dim])
    start = np.concatenate([[0], np.cumsum(CAT_SIZES[out_dim])[:-1]])
    return cat, (np.arange(len(cat)) - start[cat]).astype(np.uint16)


def outcome_values(y, ref_gt21):
    """float32 [B, 804|24]: every list of ``possible_outcome_probabilites_from`` concatenated in category order, each product
    in the reference's left-to-right float32 order."""
    y = np.asarray(y, dtype=np.float32)
    n = len(y)
    g, homref, homvar, hetvar = y[:, :21], y[:, 21], y[:, 22], y[:, 23]
    gref = g[np.arange(n), np.asarray(ref_gt21).astype(np.int64)]
    col = lambda a: a[:, None]                                                   # noqa: E731
    if y.shape[1] == 24:
        parts = [col(homref * gref), col(homvar) * g[:, HOMO_SNP_GT21], col(hetvar) * g[:, HETERO_SNP_GT21],
                 col(homvar * g[:, GT21_INSINS]), g[:, GT21_AINS:GT21_AINS + 4] * col(hetvar), col(hetvar * g[:, GT21_INSINS]),
                 col(homvar * g[:, GT21_DELDEL]), g[:, GT21_ADEL:GT21_ADEL + 4] * col(hetvar), col(hetvar * g[:, GT21_DELDEL]),
                 col(hetvar * g[:, GT21_INSDEL])]
    else:
        v1, v2 = y[:, 24:57], y[:, 57:90]
        vl0 = v1[:, 16] * v2[:, 16]
        ins = np.arange(17, 33)                  # length i -> i + index_offset
        dele = 16 - np.arange(1, 17)             # length i -> -i + index_offset
        ii, dd, idl = np.array(INSINS_PAIRS), np.array(DELDEL_PAIRS), np.array(INSDEL_PAIRS)
        parts = [col((vl0 * homref) * gref), col(vl0 * homvar) * g[:, HOMO_SNP_GT21], col(vl0 * hetvar) * g[:, HETERO_SNP_GT21],
                 (v1[:, ins] * v2[:, ins]) * col(homvar * g[:, GT21_INSINS]),
                 ((col(v1[:, 16]) * v2[:, ins])[:, :, None] * g[:, None, GT21_AINS:GT21_AINS + 4] * hetvar[:, None, None]).reshape(n, 64),
                 (v1[:, 16 + ii[:, 0]] * v2[:, 16 + ii[:, 1]]) * col(hetvar * g[:, GT21_INSINS]),
                 (v1[:, dele] * v2[:, dele]) * col(homvar * g[:, GT21_DELDEL]),
                 ((v1[:, dele] * col(v2[:, 16]))[:, :, None] * g[:, None, GT21_ADEL:GT21_ADEL + 4] * hetvar[:, None, None]).reshape(n, 64),
                 (v1[:, 16 - dd[:, 0]] * v2[:, 16 - dd[:, 1]]) * col(hetvar * g[:, GT21_DELDEL]),
                 (v1[:, 16 - idl[:, 0]] * v2[:, 16 + idl[:, 1]]) * col(hetvar * g[:, GT21_INSDEL])]
    out = np.concatenate([np.asarray(p, dtype=np.float32).reshape(n, -1) for p in parts], axis=1)
    assert out.dtype == np.float32 and out.shape[1] == sum(CAT_SIZES[y.shape[1]])
    return out


def decode_stage2(y, ref_gt21, sites=None, n_sites=None, k=16):
    """The first ``k`` entries of every listed site's attempt order: probability descending, then category, then index
    ascending, ending at (and including) homo_Ref.  Returns the dict ``Clair3_X.decode_stage2`` returns (numpy):
    cat / idx / prob / tie_mask [S, k] (padding: cat 255, idx 0, prob 0, mask 0), count [S], complete [S].
    ``tie_mask`` bit c: category c holds an entry with the same probability at this position of the order or later - the
    ``is_*`` flags ``output_from`` returns when this attempt succeeds."""
    y = np.asarray(y, dtype=np.float32)
    ref_gt21 = np.asarray(ref_gt21)
    B, out_dim = y.shape
    sites = np.arange(B) if sites is None else np.asarray(sites, dtype=np.int64)
    S = len(sites)
    n = S if n_sites is None else int(np.asarray(n_sites).reshape(-1)[0])
    E = sum(CAT_SIZES[out_dim])
    out = {"cat": np.full((S, k), PAD_CAT, dtype=np.uint8), "idx": np.zeros((S, k), dtype=np.uint16),
           "prob": np.zeros((S, k), dtype=np.float32), "tie_mask": np.zeros((S, k), dtype=np.uint16),
           "count": np.zeros(S, dtype=np.int32), "complete": np.zeros(S, dtype=np.uint8)}
    if n == 0:
        return out
    rows = sites[:n].astype(np.int64)
    vals = outcome_values(y[rows], ref_gt21[rows])
    order = np.argsort(-vals, axis=1, kind="stable")                 # ties keep slot order = (category, index) order
    sv = np.take_along_axis(vals, order, axis=1)
    slot_cat, slot_idx = category_of_slot(out_dim)
    cats = slot_cat[order]
    mask = (np.uint16(1) << cats.astype(np.uint16)).astype(np.uint16)
    for t in range(E - 2, -1, -1):                                   # OR over the rest of each run of equal probabilities
        eq = sv[:, t] == sv[:, t + 1]
        mask[eq, t] |= mask[eq, t + 1]
    ref_pos = np.argmax(order == 0, axis=1)
    count = np.minimum(ref_pos + 1, k)
    kk = min(k, E)
    valid = np.arange(kk)[None, :] < count[:, None]
    out["cat"][:n, :kk] = np.where(valid, cats[:, :kk], PAD_CAT)
    out["idx"][:n, :kk] = np.where(valid, slot_idx[order[:, :kk]], 0)
    out["prob"][:n, :kk] = np.where(valid, sv[:, :kk], np.float32(0))
    out["tie_mask"][:n, :kk] = np.where(valid, mask[:, :kk], 0)
    out["count"][:n] = count
    out["complete"][:n] = (ref_pos < k).astype(np.uint8)
    return out
