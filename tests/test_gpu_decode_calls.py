"""``c3b_decode_calls`` on the GPU: records bit-exact against the record oracle (``oracle/decode_calls_oracle.py``, which formats
to the reference's text in ``tests/test_decode_calls_cpu.py``) on the fixture rows and on seeded heavy alt_info, host and
device pointers, k in {1, 16}; ``decode.batch_output`` through the records route without the host walk; the chained call on a
side stream; edge cases and argument checks."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "decode_stage2.npz")
CALLS_GOLDEN = os.path.join(HERE, "golden", "decode_calls.npz")
_MODELS = {}


def model(out_dim):
    if out_dim not in _MODELS:
        from clair3_b200 import synth
        from clair3_b200.model import Clair3_P
        add_indel = out_dim == 90
        m = Clair3_P(add_indel_length=add_indel, predict=True, input_channels=18)
        m.to(torch.device("cuda"))
        m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in synth.pileup_state_dict(add_indel, seed=1).items()})
        _MODELS[out_dim] = m
    return _MODELS[out_dim]


def config(out_dim, **kw):
    from clair3_b200 import decode
    return decode.replay_config(pileup=out_dim == 24, add_indel_length=out_dim == 90)._replace(quality_score_for_pass=None)._replace(**kw)


CONFIGS = {"default": {}, "show_ref": {"is_show_reference": True}, "haploid_precise": {"is_haploid_precise_mode_enabled": True},
           "haploid_sensitive": {"is_haploid_sensitive_mode_enabled": True},
           "long_indel": {"enable_long_indel": True, "is_show_reference": True, "maximum_variant_length_that_need_infer": 100000},
           "qual_iupac": {"quality_score_for_pass": 12.0, "keep_iupac_bases": True}}


def pack(alts):
    bs = [a.encode() if isinstance(a, str) else bytes(a) for a in alts]
    off = np.zeros(len(bs) + 1, np.int64)
    np.cumsum([len(b) for b in bs], out=off[1:])
    return np.frombuffer(b"".join(bs), np.uint8).copy(), off


def run(m, y, ref, alts, cfg, where="cpu", k=16):
    from clair3_b200.model import CALL_DTYPE
    ab, off = pack(alts)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(where)        # noqa: E731
    out = m.decode_calls(t(y), t(ref), t(ab), t(off), cfg, k=k)
    torch.cuda.synchronize()
    out = {k_: v.cpu().numpy() for k_, v in out.items()}
    out["calls"] = out["calls"].view(CALL_DTYPE).reshape(len(y))
    return out, off


def oracle(y, ref, alts, cfg):
    from oracle import decode_calls_oracle as dco
    ab, off = pack(alts)
    return dco.decode_calls(y, ref, ab, off, cfg)


def assert_same(got, want, off):
    g, w = got["calls"], want["calls"]
    assert np.array_equal(g["status"], w["status"])
    ok = w["status"] == 0
    for name in ("dp", "support", "ref_count", "ref_len", "alt_len", "n_ad", "flags", "genotype", "printed"):
        assert np.array_equal(g[name][ok], w[name][ok]), name
    assert np.array_equal(g["prob"][ok].view(np.uint32), w["prob"][ok].view(np.uint32))
    for s in np.nonzero(ok)[0]:
        o = 2 * off[s] + 8 * s
        n = int(w["ref_len"][s] + w["alt_len"][s])
        assert got["text"][o:o + n].tobytes() == want["text"][o:o + n].tobytes(), s
        assert np.array_equal(got["ad"][o:o + w["n_ad"][s]], want["ad"][o:o + w["n_ad"][s]]), s


def fixture(out_dim):
    z = np.load(GOLDEN)
    pre = "real%d_" % out_dim
    pos = [str(p) for p in z[pre + "pos"]]
    ref = np.array([ord(p.split(":")[-1][16]) for p in pos], np.uint8)
    return z[pre + "y"], ref, [str(a) for a in z[pre + "alt"]], pos, z


def rnd(r, n, alphabet="ACGT"):
    return "".join(r.choice(list(alphabet), size=n))


def heavy_sites(n, out_dim, seed):
    """Seeded rows (softmax heads, a fifth quantised to quarters for exact ties) with heavy alt_info: up to 64 alleles, insertions
    up to 500 bases, long-indel lengths around 50, repeated keys, lowercase / IUPAC deletions and reference bases."""
    r = np.random.default_rng(seed)
    bounds = [0, 21, 24, 57, 90][: (5 if out_dim == 90 else 3)]
    y = np.empty((n, out_dim), np.float32)
    scale = r.choice([0.3, 2.0, 6.0, 15.0], size=(n, 1))
    for lo, hi in zip(bounds, bounds[1:]):
        zz = np.exp(r.standard_normal((n, hi - lo)) * scale)
        y[:, lo:hi] = zz / zz.sum(1, keepdims=True)
    q = r.random(n) < 0.2
    y[q] = (r.integers(0, 5, size=(q.sum(), out_dim)) / 4.0).astype(np.float32)
    refs = r.choice(list("ACGTACGTACGTRYKMN"), size=n)
    alts = []
    lens = [1, 2, 3, 5, 8, 14, 15, 16, 17, 30, 45, 46, 49, 50, 51, 52, 55, 56, 60, 100, 500]
    for i in range(n):
        anchor = {"R": "A", "Y": "C", "K": "G", "M": "A", "N": "A"}.get(refs[i], refs[i])
        heavy = r.random() < 0.05
        items = [("X" + b, int(r.integers(0, 40))) for b in r.choice(list("ACGT"), size=int(r.integers(0, 5)))]
        for _ in range(int(r.integers(0, 60 if heavy else 5))):
            items.append(("I" + anchor + rnd(r, int(r.choice(lens))), int(r.integers(0, 30))))
        for _ in range(int(r.integers(0, 8 if heavy else 5))):
            items.append(("D" + rnd(r, int(r.choice(lens[:-2])), "ACGT" if r.random() < 0.8 else "acgtRYN"), int(r.integers(0, 30))))
        if r.random() < 0.8:
            items.append(("R", int(r.integers(0, 50))))
        r.shuffle(items)
        depth = int(r.integers(0, 3)) if r.random() < 0.05 else int(r.integers(20, 120))
        body = " ".join("%s %d" % kv for kv in items)
        alts.append("%d-%s" % (depth, body) if body else "%d" % depth)
    return y, np.array([ord(c) for c in refs], np.uint8), alts


@pytest.mark.parametrize("name", list(CONFIGS))
@pytest.mark.parametrize("out_dim", [24, 90])
def test_fixture_rows_bit_exact(out_dim, name):
    y, ref, alts, _, _ = fixture(out_dim)
    cfg = config(out_dim, **CONFIGS[name])
    want = oracle(y, ref, alts, cfg)
    for where, k in (("cpu", 16), ("cuda", 1)):
        got, off = run(model(out_dim), y, ref, alts, cfg, where, k)
        assert_same(got, want, off)


@pytest.mark.parametrize("name", list(CONFIGS))
@pytest.mark.parametrize("out_dim", [24, 90])
def test_targeted_fixture_bit_exact_and_reference_text(out_dim, name):
    """tests/golden/decode_calls.npz (minted from the reference): the records of all rows in one batch are bit-exact to the
    oracle (statuses included), and batch_output on the GPU gives the reference's rows, or raises its exception per row."""
    from clair3_b200 import decode
    z = np.load(CALLS_GOLDEN)
    pre = "c%d_" % out_dim
    y, pos, alts = z[pre + "y"], [str(p) for p in z[pre + "pos"]], [str(a) for a in z[pre + "alt"]]
    ref = np.array([ord(p.split(":")[-1][16]) for p in pos], np.uint8)
    cfg = config(out_dim, **CONFIGS[name])
    want = oracle(y, ref, alts, cfg)
    for where, k in (("cuda", 16), ("cpu", 1)):
        got, off = run(model(out_dim), y, ref, alts, cfg, where, k)
        assert_same(got, want, off)
    texts, excs = z[pre + "text_" + name], z[pre + "exc_" + name]
    ok = np.nonzero(excs == "")[0]
    text = decode.batch_output(model(out_dim), [pos[i] for i in ok], [alts[i] for i in ok], y[ok], cfg)
    assert text == "".join(str(texts[i]) for i in ok)
    if name == "default":
        for i in np.nonzero(excs != "")[0]:
            with pytest.raises(Exception) as e:
                decode.batch_output(model(out_dim), [pos[i]], [alts[i]], y[i:i + 1], cfg)
            assert type(e.value).__name__ == str(excs[i]), (i, alts[i])


@pytest.mark.parametrize("out_dim", [24, 90])
def test_seeded_heavy_sites_bit_exact(out_dim):
    y, ref, alts = heavy_sites(20_000, out_dim, seed=11 + out_dim)
    for cfg in (config(out_dim), config(out_dim, **CONFIGS["long_indel"])):
        want = oracle(y, ref, alts, cfg)
        assert (want["calls"]["status"] == 0).all() and want["calls"]["printed"].mean() > 0.3
        for where, k in (("cuda", 16), ("cpu", 1)):
            got, off = run(model(out_dim), y, ref, alts, cfg, where, k)
            assert_same(got, want, off)


@pytest.mark.parametrize("out_dim", [24, 90])
def test_batch_output_records_route_without_host_walk(out_dim, monkeypatch):
    from clair3_b200 import decode

    def no_walk(*a, **k):
        raise AssertionError("the host walk ran")

    monkeypatch.setattr(decode, "output_from_ranked", no_walk)
    y, _, alts, pos, z = fixture(out_dim)
    for name, kw in CONFIGS.items():
        for k in (1, 16):
            text = decode.batch_output(model(out_dim), pos, alts, y, config(out_dim, **kw), k=k)
            assert text == z["real%d_text_%s" % (out_dim, name)].item(), (name, k)


@pytest.mark.parametrize("out_dim", [24, 90])
def test_side_stream_chain_equals_host_call(out_dim):
    from clair3_b200.model import CALL_DTYPE
    y, ref, alts = heavy_sites(3000, out_dim, seed=3)
    cfg = config(out_dim, is_show_reference=True)
    host, off = run(model(out_dim), y, ref, alts, cfg, "cpu", 16)
    ab, off = pack(alts)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        dev = model(out_dim).decode_calls(torch.from_numpy(y).cuda(), torch.from_numpy(ref).cuda(), torch.from_numpy(ab).cuda(),
                                          torch.from_numpy(off).cuda(), cfg, k=16)
        got = {k: v.to("cpu", non_blocking=True) for k, v in dev.items()}
    s.synchronize()
    got = {k: v.numpy() for k, v in got.items()}
    got["calls"] = got["calls"].view(CALL_DTYPE).reshape(len(y))
    assert_same(got, host, off)


def test_edge_cases():
    from clair3_b200 import decode
    m = model(90)
    cfg = config(90, is_show_reference=True)
    y = np.zeros((40, 90), np.float32)                         # every site an early-out reference call
    y[:, 21] = 0.9
    y[:, 0] = 0.8
    y[:, 40] = y[:, 73] = 0.9
    ref = np.full(40, ord("A"), np.uint8)
    alts = ["%d-XC 3 R %d" % (30 + i, i) for i in range(40)]
    got, off = run(m, y, ref, alts, cfg)
    assert (got["calls"]["flags"] == 1).all() and (got["calls"]["printed"] == 1).all()
    assert_same(got, oracle(y, ref, alts, cfg), off)
    empty, _ = run(m, y[:0], ref[:0], [], cfg)
    assert len(empty["calls"]) == 0
    pos = ["chr1:%d:%s" % (i, "A" * 33) for i in range(3)]
    yy = np.zeros((3, 90), np.float32)
    yy[:, 22] = yy[:, 4] = 0.9                                  # homo-variant C: the walk reads the keys
    yy[:, 40] = yy[:, 73] = 0.9
    big = ["30-XC 4611686018427387904 R 1", "30-XC 4611686018427387905", "30-XC 9300000000000000000", "30-XC 12345678901234567890123"]
    got, off = run(m, yy[:1].repeat(4, 0), np.full(4, ord("A"), np.uint8), big, cfg)
    assert list(got["calls"]["status"]) == [0, 4, 4, 4]
    assert_same(got, oracle(yy[:1].repeat(4, 0), np.full(4, ord("A"), np.uint8), big, cfg), off)
    for bad, exc in (("x-XC 3", ValueError), ("30-XC three", ValueError), ("30-X 3", IndexError), ("30- 3", IndexError)):
        with pytest.raises(exc):
            decode.batch_output(m, pos, ["30-XC 5", bad, "30-XC 5"], yy, cfg)


def test_bad_arguments_raise_cleanly():
    from clair3_b200._ffi import C3BError, ffi, lib
    m = model(24)
    y, ref, alts = heavy_sites(10, 24, seed=2)
    ab, off = pack(alts)
    cfg = config(24)
    with pytest.raises(C3BError, match="k must"):
        m.decode_calls(y, ref, ab, off, cfg, k=0)
    with pytest.raises(C3BError, match="add_indel_length"):
        m.decode_calls(y, ref, ab, off, config(90))
    with pytest.raises(C3BError, match="alt_offsets"):
        m.decode_calls(y, ref, ab, off[:-1], cfg)
    with pytest.raises(C3BError, match="ref_base"):
        m.decode_calls(torch.from_numpy(y).cuda(), torch.from_numpy(ref), ab, off, cfg)
    calls = ffi.new("c3b_call[10]")
    text = ffi.new("char[]", 2 * len(ab) + 80)
    ad = ffi.new("int64_t[]", 2 * len(ab) + 80)
    c = ffi.cast
    args = lambda o, k=16, bits=0: (m._handle, c("float *", y.ctypes.data), c("uint8_t *", ref.ctypes.data), 10,  # noqa: E731
                                    c("char *", ab.ctypes.data), c("int64_t *", o.ctypes.data), len(ab), bits, 50, k, 0, calls,
                                    text, ad, ffi.NULL)
    assert lib().c3b_decode_calls(*args(off, k=1025)) != 0
    assert b"k must" in ffi.string(lib().c3b_last_error())
    assert lib().c3b_decode_calls(*args(off, bits=64)) != 0
    assert b"config" in ffi.string(lib().c3b_last_error())
    bad = off.copy()
    bad[3] = bad[5] + 1
    assert lib().c3b_decode_calls(*args(bad)) != 0
    assert b"alt_offsets" in ffi.string(lib().c3b_last_error())
    assert lib().c3b_decode_calls(ffi.NULL, *args(off)[1:]) != 0
    assert lib().c3b_decode_calls(*args(off)) == 0
