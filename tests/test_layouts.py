"""CPU model of the HBM layouts and the shifted-view index arithmetic the CUDA convolution kernel relies on
(clair3_b200/csrc/pconv_tc.cu, c3b_internal.h: c3b_planar_geom / c3b_parity_offset; DESIGN.md 2).

The kernel never gathers: a 3x3 tap is the SAME zero-padded planar image (stride 1) or one of four parity planes (stride 2)
viewed a constant number of slots later.  These tests restate that claim in numpy and check it against the oracle's
im2col convolution (oracle/clair3_oracle.py:_im2col3x3, itself pinned to the reference by tests/test_oracle.py), on ragged
shapes including the network's real 89x33 / 45x17 / 23x9 / 12x5 levels.
"""
import numpy as np
import pytest

from oracle import clair3_oracle as orc


def planar_geom(batch, h, w):
    """Mirror of c3b_planar_geom."""
    wp = w + 2
    s = (h + 2) * wp
    g = (wp + 1 + 7) // 8 * 8
    t = batch * s
    p = g + (t + 511) // 512 * 512 + g
    return dict(h=h, w=w, wp=wp, s=s, g=g, t=t, p=p)


def to_planar(x, geo):
    """x: [B,C,H,W] -> planar padded [C][P] (the kernel additionally groups channels by 8: irrelevant to the slot arithmetic)."""
    b, c, h, w = x.shape
    out = np.zeros((c, geo["p"]), dtype=x.dtype)
    for bi in range(b):
        for hh in range(h):
            base = geo["g"] + bi * geo["s"] + (hh + 1) * geo["wp"] + 1
            out[:, base:base + w] = x[bi, :, hh, :]
    return out


def to_parity_planes(x, geo_out):
    """x: [B,C,H,W] (the stride-2 conv's input) -> four planes [4][C][P'] in the OUTPUT level's geometry: padded pixel
    (hp, wp) = (h+1, w+1) lives in plane (hp&1)*2 + (wp&1) at slot (hp>>1, wp>>1) (mirror of c3b_parity_offset)."""
    b, c, h, w = x.shape
    out = np.zeros((4, c, geo_out["p"]), dtype=x.dtype)
    for bi in range(b):
        for hh in range(h):
            for ww in range(w):
                hp, wp = hh + 1, ww + 1
                plane = (hp & 1) * 2 + (wp & 1)
                slot = geo_out["g"] + bi * geo_out["s"] + ((hp >> 1) + 1) * geo_out["wp"] + ((wp >> 1) + 1)
                out[plane, :, slot] = x[bi, :, hh, ww]
    return out


def real_slots(geo, batch):
    idx = []
    for bi in range(batch):
        for hh in range(geo["h"]):
            for ww in range(geo["w"]):
                idx.append(geo["g"] + bi * geo["s"] + (hh + 1) * geo["wp"] + (ww + 1))
    return np.asarray(idx)


def conv_reference(x, w, stride):
    cols, ho, wo = orc._im2col3x3(x, stride)
    return (cols @ w.reshape(w.shape[0], -1).T).transpose(0, 3, 1, 2)       # [B,Cout,Ho,Wo]


@pytest.mark.parametrize("shape", [(2, 3, 12, 5), (1, 4, 23, 9), (3, 2, 7, 4), (1, 1, 1, 1)])
def test_stride1_conv_is_nine_shifted_views_of_one_planar_image(shape):
    r = np.random.default_rng(sum(shape))
    b, c, h, w = shape
    x = r.standard_normal(shape)
    wt = r.standard_normal((5, c, 3, 3))
    geo = planar_geom(b, h, w)
    img = to_planar(x, geo)
    slots = real_slots(geo, b)
    acc = np.zeros((5, len(slots)))
    for dh in range(3):
        for dw in range(3):
            shift = (dh - 1) * geo["wp"] + (dw - 1)       # the kernel loads a (wp+1)-slot halo and uses dh*wp + dw
            acc += wt[:, :, dh, dw] @ img[:, slots + shift]
    ref = conv_reference(x, wt, 1).transpose(1, 0, 2, 3).reshape(5, -1)
    assert np.abs(acc - ref).max() < 1e-10
    # the halo never leaves the plane: guards are at least wp + 1 slots
    assert geo["g"] >= geo["wp"] + 1 and slots.min() - (geo["wp"] + 1) >= 0 and slots.max() + geo["wp"] + 1 < geo["p"]


@pytest.mark.parametrize("shape", [(2, 3, 89, 33), (1, 2, 45, 17), (2, 2, 23, 9), (1, 3, 55, 33), (2, 1, 5, 3), (1, 1, 1, 1)])
def test_stride2_conv_is_shifted_views_of_four_parity_planes(shape):
    r = np.random.default_rng(sum(shape) + 1)
    b, c, h, w = shape
    x = r.standard_normal(shape)
    wt = r.standard_normal((4, c, 3, 3))
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    geo = planar_geom(b, ho, wo)                           # planes live in the OUTPUT level's geometry
    planes = to_parity_planes(x, geo)
    slots = real_slots(geo, b)
    acc = np.zeros((4, len(slots)))
    for dh in range(3):
        for dw in range(3):
            plane = (dh & 1) * 2 + (dw & 1)
            shift = (dh >> 1) * geo["wp"] + (dw >> 1)
            acc += wt[:, :, dh, dw] @ planes[plane][:, slots + shift]
    ref = conv_reference(x, wt, 2).transpose(1, 0, 2, 3).reshape(4, -1)
    assert ref.shape[1] == len(slots)
    assert np.abs(acc - ref).max() < 1e-10
    assert slots.max() + geo["wp"] + 1 < geo["p"]          # the kernel reads up to wp + 1 slots past a macro-tile


def test_planar_borders_stay_zero_and_sites_do_not_alias():
    geo = planar_geom(3, 12, 5)
    x = np.ones((3, 2, 12, 5))
    img = to_planar(x, geo)
    slots = real_slots(geo, 3)
    assert len(set(slots.tolist())) == 3 * 12 * 5
    mask = np.ones(geo["p"], dtype=bool)
    mask[slots] = False
    assert np.all(img[:, mask] == 0) and np.all(img[:, slots] == 1)
    # plane pitch covers the rounded-up slot range the macro-tiles walk (multiples of 512 slots) plus both guards
    assert geo["p"] % 8 == 0 and geo["p"] >= 2 * geo["g"] + geo["t"]


def test_kgroup_planar_flatten_order_matches_reference_flatten():
    """h2 / spp are stored [K/8][rows][8]; k must follow the reference's flatten order (model.py:135: [B,33,320] -> 10560)."""
    b, t, f = 3, 33, 320
    h = np.arange(b * t * f, dtype=np.int64).reshape(b, t, f)
    flat = h.reshape(b, t * f)                              # the reference's flatten
    planar = np.zeros((t * f // 8, b, 8), dtype=np.int64)
    for bi in range(b):
        for tt in range(t):
            for d in range(2):
                for j in range(160):
                    k = tt * 320 + d * 160 + j              # DESIGN.md 2: k = t*320 + dir*160 + j
                    planar[k >> 3, bi, k & 7] = h[bi, tt, d * 160 + j]
    back = planar.transpose(1, 0, 2).reshape(b, t * f)
    assert np.array_equal(back, flat)
