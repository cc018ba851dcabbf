"""Seeded synthetic checkpoints and candidate-site batches for the Clair3 hot path.

No released ``.pt`` checkpoint or BAM exists offline, so parity tests, golden fixtures and
``bench.py`` all draw weights and inputs from here.  Everything is generated with
``numpy.random.Generator(PCG64(seed))`` so the very same arrays are rebuilt on the GPU machine
without shipping multi-megabyte fixtures.

State-dict key names / shapes follow the reference modules
(``clair3/model.py:96-128`` for ``Clair3_P``, ``clair3/model.py:317-368`` for ``Clair3_F``);
input layouts follow ``shared/param_p.py:32-36`` ([33,18] per site) and
``shared/param_f.py:29-30`` ([depth,33,C] per site, values in [-100,100]).
"""
from __future__ import annotations

import numpy as np

P_POSITIONS = 33
P_CHANNELS = 18
F_WIDTH = 33
HEAD_DIMS = (21, 3, 33, 33)


def _rng(seed):
    return np.random.Generator(np.random.PCG64(seed))


def _normal(r, shape, std):
    return (r.standard_normal(shape) * std).astype(np.float32)


def pileup_state_dict(add_indel_length=False, channels=P_CHANNELS, seed=0):
    """Trained-like synthetic ``Clair3_P`` state_dict (numpy fp32), reference key order."""
    r = _rng(seed)
    sd = {}
    h1, h2 = 128, 160
    for name, inp, hid, s_ih, s_hh in (("LSTM1", channels, h1, 0.05, 0.11),
                                       ("LSTM2", 2 * h1, h2, 0.09, 0.11)):
        for suffix in ("", "_reverse"):
            sd[f"{name}.weight_ih_l0{suffix}"] = _normal(r, (4 * hid, inp), s_ih)
            sd[f"{name}.weight_hh_l0{suffix}"] = _normal(r, (4 * hid, hid), s_hh)
            sd[f"{name}.bias_ih_l0{suffix}"] = _normal(r, (4 * hid,), 0.1)
            sd[f"{name}.bias_hh_l0{suffix}"] = _normal(r, (4 * hid,), 0.1)
    sd["L4.weight"] = _normal(r, (128, 2 * h2 * P_POSITIONS), 3.0 / np.sqrt(2 * h2 * P_POSITIONS))
    sd["L4.bias"] = _normal(r, (128,), 0.1)
    heads = [("L5_1", "Y_gt21_logits", 21), ("L5_2", "Y_genotype_logits", 3)]
    if add_indel_length:
        heads += [("L5_3", "Y_indel_length_logits_1", 33), ("L5_4", "Y_indel_length_logits_2", 33)]
    # reference registration order: L5_1, L5_2, Y_gt21, Y_genotype, then L5_3, L5_4, Y_indel_1, Y_indel_2
    for l5, _, _ in heads[:2]:
        sd[f"{l5}.weight"] = _normal(r, (128, 128), 1.5 / np.sqrt(128))
        sd[f"{l5}.bias"] = _normal(r, (128,), 0.1)
    for _, y, n in heads[:2]:
        sd[f"{y}.weight"] = _normal(r, (n, 128), 4.0 / np.sqrt(128))
        sd[f"{y}.bias"] = _normal(r, (n,), 0.2)
    for l5, _, _ in heads[2:]:
        sd[f"{l5}.weight"] = _normal(r, (128, 128), 1.5 / np.sqrt(128))
        sd[f"{l5}.bias"] = _normal(r, (128,), 0.1)
    for _, y, n in heads[2:]:
        sd[f"{y}.weight"] = _normal(r, (n, 128), 4.0 / np.sqrt(128))
        sd[f"{y}.bias"] = _normal(r, (n,), 0.2)
    return sd


def _conv_bn(r, sd, conv_key, bn_key, cout, cin):
    sd[f"{conv_key}.weight"] = _normal(r, (cout, cin, 3, 3), np.sqrt(2.0 / (9 * cin)))
    sd[f"{conv_key}.bias"] = _normal(r, (cout,), 0.05)
    sd[f"{bn_key}.weight"] = r.uniform(0.5, 1.5, cout).astype(np.float32)
    sd[f"{bn_key}.bias"] = _normal(r, (cout,), 0.1)
    sd[f"{bn_key}.running_mean"] = _normal(r, (cout,), 0.1)
    sd[f"{bn_key}.running_var"] = r.uniform(0.5, 1.5, cout).astype(np.float32)
    sd[f"{bn_key}.num_batches_tracked"] = np.array(1234, dtype=np.int64)


def fa_state_dict(add_indel_length=True, channels=8, seed=0):
    """Trained-like synthetic ``Clair3_F`` state_dict (numpy), BN running stats non-trivial."""
    r = _rng(seed + 1000)
    sd = {}
    _conv_bn(r, sd, "conv1.conv", "conv1.bn", 64, channels)
    for blk, stem, cin, c in (("res_block1", "conv3", 64, 64), ("res_block2", "conv5", 128, 128),
                              ("res_block3", None, 256, 256)):
        _conv_bn(r, sd, f"{blk}.0.conv1", f"{blk}.0.bn1", c, c)
        _conv_bn(r, sd, f"{blk}.0.conv2", f"{blk}.0.bn2", c, c)
        if stem is not None:
            _conv_bn(r, sd, f"{stem}.conv", f"{stem}.bn", 2 * c, c)
    # re-order to the reference's registration order (conv1, res_block1, conv3, res_block2, conv5, res_block3)
    order = []
    for prefix in ("conv1.", "res_block1.", "conv3.", "res_block2.", "conv5.", "res_block3."):
        order += [k for k in sd if k.startswith(prefix)]
    sd = {k: sd[k] for k in order}
    sd["L4.weight"] = _normal(r, (256, 3584), 0.35 / np.sqrt(3584))
    sd["L4.bias"] = _normal(r, (256,), 0.1)
    heads = [("L5_1", "Y_gt21_logits", 21), ("L5_2", "Y_genotype_logits", 3)]
    if add_indel_length:
        heads += [("L5_3", "Y_indel_length_logits_1", 33), ("L5_4", "Y_indel_length_logits_2", 33)]
    for l5, _, _ in heads[:2]:
        sd[f"{l5}.weight"] = _normal(r, (128, 256), 1.5 / np.sqrt(256))
        sd[f"{l5}.bias"] = _normal(r, (128,), 0.1)
    for _, y, n in heads[:2]:
        sd[f"{y}.weight"] = _normal(r, (n, 128), 4.0 / np.sqrt(128))
        sd[f"{y}.bias"] = _normal(r, (n,), 0.2)
    for l5, _, _ in heads[2:]:
        sd[f"{l5}.weight"] = _normal(r, (128, 256), 1.5 / np.sqrt(256))
        sd[f"{l5}.bias"] = _normal(r, (128,), 0.1)
    for _, y, n in heads[2:]:
        sd[f"{y}.weight"] = _normal(r, (n, 128), 4.0 / np.sqrt(128))
        sd[f"{y}.bias"] = _normal(r, (n,), 0.2)
    return sd


def pileup_inputs(batch, seed=0, realistic=True, dtype=np.int32):
    """[batch,33,18] candidate-site count tensors.

    ``realistic=False`` is SURVEY §8(d)'s uniform draw in [-60,60]; ``realistic=True`` mimics
    ``src/clair3_pileup.c:286,370-371``: non-negative per-strand counts, the reference-base
    channel holding minus the sum of the ACGT counts, depth ~ Poisson(40) with a few deep sites.
    """
    r = _rng(seed + 7)
    if not realistic:
        return r.integers(-60, 61, size=(batch, P_POSITIONS, P_CHANNELS)).astype(dtype)
    x = np.zeros((batch, P_POSITIONS, P_CHANNELS), dtype=np.int64)
    depth = r.poisson(40, size=(batch, 1)).astype(np.int64)
    deep = r.random((batch, 1)) < 0.03
    depth = np.where(deep, depth * 3, depth)            # a few sites deeper than 1.5*144/… range
    depth = np.broadcast_to(depth, (batch, P_POSITIONS))
    fwd = r.binomial(depth, 0.5)
    rev = depth - fwd
    ref = r.integers(0, 4, size=(batch, P_POSITIONS))
    err = r.random((batch, P_POSITIONS)) < 0.15
    alt = (ref + r.integers(1, 4, size=ref.shape)) % 4
    alt_frac = np.where(err, r.uniform(0.05, 0.6, size=ref.shape), 0.0)
    bi = np.arange(batch)[:, None]
    pi = np.arange(P_POSITIONS)[None, :]
    for strand_off, cnt in ((0, fwd), (9, rev)):
        a = np.floor(cnt * alt_frac).astype(np.int64)
        x[bi, pi, strand_off + alt] += a
        x[bi, pi, strand_off + ref] -= cnt             # reference channel: minus the ACGT total
        ind = r.random((batch, P_POSITIONS)) < 0.05
        x[bi, pi, strand_off + 4] += np.where(ind, r.integers(0, 6, size=ref.shape), 0)
        x[bi, pi, strand_off + 6] += np.where(ind, r.integers(0, 6, size=ref.shape), 0)
    x[:, :, 17] = r.integers(0, 3, size=(batch, P_POSITIONS))
    if np.dtype(dtype) == np.int8:
        x = ((x + 128) % 256) - 128                    # CreateTensorPileupFromCffi.py:447 narrows to int8
    return x.astype(dtype)


def fa_inputs(batch, depth=89, channels=8, seed=0, realistic=True):
    """[batch,depth,33,channels] int8 haplotype read images (values in [-100,100])."""
    r = _rng(seed + 13)
    if not realistic:
        return r.integers(-100, 101, size=(batch, depth, F_WIDTH, channels)).astype(np.int8)
    x = r.choice(np.array([-100, -50, -30, 0, 0, 0, 25, 50, 75, 100], dtype=np.int8),
                 size=(batch, depth, F_WIDTH, channels))
    x[..., 3] = r.integers(0, 101, size=x.shape[:-1])   # mapping quality channel
    x[..., 4] = r.integers(0, 101, size=x.shape[:-1])   # base quality channel
    if channels > 8:
        x[..., 8] = r.integers(0, 40, size=x.shape[:-1])  # dwell: small non-negative ints
    nreads = r.integers(10, depth + 1, size=batch)
    mask = np.arange(depth)[None, :] < nreads[:, None]  # rows beyond read depth are all-zero
    x = x * mask[:, :, None, None]
    return x.astype(np.int8)


def out_dim(add_indel_length):
    return 90 if add_indel_length else 24
