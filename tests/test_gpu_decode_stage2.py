"""``c3b_decode_stage2`` on the GPU: bit-exact against the numpy oracle (``oracle/decode_stage2_oracle.py``, itself pinned to
the reference's own ``output_from`` walk by ``tests/test_decode_stage2_cpu.py``) on the fixture rows and on seeded rows, for
both output widths, k in {1, 16, 1024}, host and device pointers, and chained on stage 1's ``nonref_idx`` / ``n_nonref``;
the host decoder on the real stages against the reference's ``batch_output`` text; edge cases and argument checks."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "decode_stage2.npz")
_MODELS = {}


def model(out_dim):
    if out_dim not in _MODELS:
        from clair3_b200 import synth
        from clair3_b200.model import Clair3_P
        add_indel = out_dim == 90
        m = Clair3_P(add_indel_length=add_indel, predict=True, input_channels=18)
        m.to(torch.device("cuda"))
        m.eval()
        m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in synth.pileup_state_dict(add_indel, seed=1).items()})
        _MODELS[out_dim] = m
    return _MODELS[out_dim]


def seeded_rows(n, out_dim, seed):
    """Softmax heads at mixed temperatures, plus rows quantised to quarters (exact ties, zeros, 0.5)."""
    r = np.random.default_rng(seed)
    bounds = [0, 21, 24, 57, 90][: (5 if out_dim == 90 else 3)]
    y = np.empty((n, out_dim), dtype=np.float32)
    scale = r.choice([0.3, 2.0, 6.0, 15.0], size=(n, 1))
    for lo, hi in zip(bounds, bounds[1:]):
        z = r.standard_normal((n, hi - lo)) * scale
        z = np.exp(z - z.max(1, keepdims=True))
        y[:, lo:hi] = z / z.sum(1, keepdims=True)
    q = r.random(n) < 0.2
    y[q] = (r.integers(0, 5, size=(q.sum(), out_dim)) / 4.0).astype(np.float32)
    gt = r.choice(np.array([0, 4, 7, 9], dtype=np.uint8), size=n)
    return y, gt


def as_numpy(d):
    out = {k: v.cpu().numpy() for k, v in d.items()}
    out["idx"] = out["idx"].view(np.uint16)
    out["tie_mask"] = out["tie_mask"].view(np.uint16)
    return out


def assert_same(got, want):
    for name in ("count", "complete", "cat", "idx", "tie_mask"):
        assert np.array_equal(got[name], want[name]), name
    assert np.array_equal(got["prob"].view(np.uint32), want["prob"].view(np.uint32))


def run(m, y, gt, where, sites=None, n_sites=None, k=16):
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(where)    # noqa: E731
    got = m.decode_stage2(t(y), t(gt), sites=t(sites), n_sites=t(n_sites), k=k)
    torch.cuda.synchronize()
    return as_numpy(got)


def fixture_rows(out_dim):
    from clair3_b200 import decode
    z = np.load(GOLDEN)
    pos = z["real%d_pos" % out_dim]
    gt_real = np.array([decode.GT21_OF_BASE[decode.BASE2ACGT[str(p).split(":")[-1][16]]] for p in pos], dtype=np.uint8)
    return (np.concatenate([z["seq_y%d" % out_dim], z["real%d_y" % out_dim]]),
            np.concatenate([z["seq_gt%d" % out_dim], gt_real]))


@pytest.mark.parametrize("k", [1, 16, 1024])
@pytest.mark.parametrize("where", ["cuda", "cpu"])
@pytest.mark.parametrize("out_dim", [24, 90])
def test_fixture_rows_bit_exact(out_dim, where, k):
    from oracle import decode_stage2_oracle as dec2
    y, gt = fixture_rows(out_dim)
    assert_same(run(model(out_dim), y, gt, where, k=k), dec2.decode_stage2(y, gt, k=k))
    # a site list in scrambled order with repeats
    sites = np.random.default_rng(k).integers(0, len(y), size=333).astype(np.int32)
    assert_same(run(model(out_dim), y, gt, where, sites=sites, k=k), dec2.decode_stage2(y, gt, sites=sites, k=k))


@pytest.mark.parametrize("out_dim", [24, 90])
def test_seeded_rows_bit_exact(out_dim):
    from oracle import decode_stage2_oracle as dec2
    y, gt = seeded_rows(100_000, out_dim, seed=out_dim)
    m = model(out_dim)
    got = run(m, y, gt, "cuda", k=16)
    want = dec2.decode_stage2(y, gt, k=16)
    assert_same(got, want)
    assert 0 < want["complete"].mean() < 1 and (np.bitwise_count(want["tie_mask"]) > 1).any()
    ys, gs = y[:4000], gt[:4000]
    assert_same(run(m, ys, gs, "cuda", k=1024), dec2.decode_stage2(ys, gs, k=1024))
    assert_same(run(m, ys, gs, "cpu", k=1), dec2.decode_stage2(ys, gs, k=1))


@pytest.mark.parametrize("out_dim", [24, 90])
def test_chains_on_stage1_on_one_stream(out_dim):
    """Stage 1's device outputs feed stage 2 directly on a side stream, with no host synchronisation in between."""
    from oracle import decode_oracle as dec1
    from oracle import decode_stage2_oracle as dec2
    y, gt = seeded_rows(3000, out_dim, seed=7 + out_dim)
    y[::3, 21] = np.float32(0.9)                                       # plenty of early-out rows to skip
    y[::3, :21] = np.float32(0.01)
    y[np.arange(0, 3000, 3), gt[::3]] = np.float32(0.8)
    if out_dim == 90:
        y[::3, 24 + 16] = y[::3, 57 + 16] = np.float32(0.9)
    m = model(out_dim)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        yd, gd = torch.from_numpy(y).cuda(), torch.from_numpy(gt).cuda()
        s1 = m.decode_stage1(yd, gd)
        s2 = m.decode_stage2(yd, gd, sites=s1["nonref_idx"], n_sites=s1["n_nonref"], k=16)
    s.synchronize()
    w1 = dec1.decode_stage1(y, gt)
    n = int(w1["n_nonref"][0])
    assert 0 < n < 3000 and int(s1["n_nonref"].item()) == n
    got = as_numpy(s2)
    want = dec2.decode_stage2(y, gt, sites=np.concatenate([w1["nonref_idx"], np.zeros(3000 - n, np.int32)]), n_sites=n, k=16)
    assert_same(got, want)
    assert (got["count"][n:] == 0).all() and (got["cat"][n:] == 255).all()


@pytest.mark.parametrize("out_dim", [24, 90])
def test_batch_output_with_gpu_stages_equals_reference_text(out_dim):
    from clair3_b200 import decode
    z = np.load(GOLDEN)
    pre = "real%d_" % out_dim
    for name, kw in (("default", {}), ("show_ref", {"is_show_reference": True}),
                     ("haploid_precise", {"is_haploid_precise_mode_enabled": True}),
                     ("haploid_sensitive", {"is_haploid_sensitive_mode_enabled": True}),
                     ("long_indel", {"enable_long_indel": True, "is_show_reference": True,
                                     "maximum_variant_length_that_need_infer": 100000}),
                     ("qual_iupac", {"quality_score_for_pass": 12.0, "keep_iupac_bases": True})):
        base = decode.replay_config(pileup=out_dim == 24, add_indel_length=out_dim == 90)._replace(quality_score_for_pass=None)
        cfg = base._replace(**kw)
        for k in (1, 16):
            text = decode.batch_output(model(out_dim), list(z[pre + "pos"]), list(z[pre + "alt"]), z[pre + "y"], cfg, k=k)
            assert text == z[pre + "text_" + name].item(), (name, k)


def test_empty_batch_and_zero_site_count():
    m = model(90)
    y, gt = seeded_rows(50, 90, seed=1)
    for where in ("cuda", "cpu"):
        empty = run(m, y[:0], gt[:0], where)
        assert empty["cat"].shape == (0, 16) and empty["count"].shape == (0,)
        none_listed = run(m, y, gt, where, sites=np.arange(50, dtype=np.int32), n_sites=np.zeros(1, np.int32))
        assert (none_listed["count"] == 0).all() and (none_listed["cat"] == 255).all() and (none_listed["complete"] == 0).all()
        no_sites = run(m, y, gt, where, sites=np.zeros(0, np.int32))
        assert no_sites["count"].shape == (0,)


def test_bad_arguments_raise_cleanly():
    from clair3_b200._ffi import C3BError, ffi, lib
    m = model(24)
    y, gt = seeded_rows(10, 24, seed=2)
    yd, gd = torch.from_numpy(y).cuda(), torch.from_numpy(gt).cuda()
    for k in (0, 1025, -3, 2.5):
        with pytest.raises(C3BError, match="k must"):
            m.decode_stage2(yd, gd, k=k)
    with pytest.raises(C3BError, match="float32"):
        m.decode_stage2(torch.zeros((10, 90), device="cuda"), gd)
    with pytest.raises(C3BError, match="ref_gt21"):
        m.decode_stage2(yd, gd[:5])
    with pytest.raises(C3BError, match="sites"):
        m.decode_stage2(yd, gd, sites=torch.zeros(3, dtype=torch.int32))              # host list for device rows
    with pytest.raises(C3BError, match="out of range"):
        m.decode_stage2(torch.from_numpy(y), torch.from_numpy(gt), sites=torch.tensor([0, 10], dtype=torch.int32))
    # the C-ABI checks its own arguments too
    out = [ffi.new("uint8_t[16]"), ffi.new("uint16_t[16]"), ffi.new("float[16]"), ffi.new("uint16_t[16]"), ffi.new("int32_t[1]"),
           ffi.new("uint8_t[1]")]
    yh = ffi.cast("float *", y.ctypes.data)
    gh = ffi.cast("uint8_t *", gt.ctypes.data)
    assert lib().c3b_decode_stage2(m._handle, yh, gh, 10, ffi.NULL, ffi.NULL, 1, 2000, 0, *out, ffi.NULL) != 0
    assert b"k must" in ffi.string(lib().c3b_last_error())
    assert lib().c3b_decode_stage2(m._handle, yh, gh, 10, ffi.NULL, ffi.NULL, 11, 16, 0, *out, ffi.NULL) != 0
    assert b"max_sites" in ffi.string(lib().c3b_last_error())
    assert lib().c3b_decode_stage2(ffi.NULL, yh, gh, 10, ffi.NULL, ffi.NULL, 1, 16, 0, *out, ffi.NULL) != 0
    assert lib().c3b_decode_stage2(m._handle, yh, gh, 10, ffi.NULL, ffi.NULL, 1, 16, 0, *out, ffi.NULL) == 0
    assert out[0][0] != 255 and out[4][0] >= 1
