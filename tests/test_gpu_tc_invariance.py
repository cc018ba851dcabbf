"""Per-site bit invariance of the fp16 tensor-core forward (option ``precision = 0``, the production path) on an H100
(``pytest -m gpu``): a site's output row must not depend on anything but the site and the model's weights.  Everything is
compared with ``torch.equal``, never with a tolerance.

Why it can hold: every site is one N column of ``wgmma.m64nNk16`` with the same K order whatever N is; the LSTM cell math runs
per thread; proj2 and the convolutions accumulate the whole of K in one CTA in a fixed order; L4 splits K into a count of
slices that depends on K alone (``c3b_launch_tail``: 15 x 11 k-chunks for the pileup net, 14 x 4 for full alignment), and
the heads kernel adds the partials in split order with per-site arithmetic that is the same for its 8- and 16-site groups and
for either head-pair layout.  An L4 split count taken from the number of tiles and the device's SM count made a site's
probabilities change with the chunk it shared (``chunk_sites`` 2600 / 4096 below) and with the card.

What must not matter, on both networks:
* neighbours and position: sub-batches, repeats and permutations at the batch edges where the kernels change shape (128-site
  tiles; the heads' 8 / 16-site groups at 512; the 1024-site pileup and 256-site full-alignment chunks; the 4-head kernel's
  pair layout at 2200 pileup sites in one chunk);
* ``chunk_sites`` from 1 to 8192, and the contiguous shards of ``sharding.site_range`` for 2, 3, 5 and 8 ranks;
* the call shape: host tensors (latency mode, another automatic LSTM tile), ``forward_into``, ``forward_async`` on several
  streams, ``predict_stream``, ``forward_windows`` against the host-gathered windows, 8 concurrent streams, two models on two
  host threads;
* kernel variants ``lstm_tile`` x ``lstm_wg`` and the input dtype (int8 / int32 / float32 holding the same values);
* a 51 200-site single chunk, whose 2.2 G-element pre-gate buffer needs 64-bit offsets;
* the full-alignment workspace's history of depths and capacities (each call against a fresh model);
* and end to end, ``chunk_sites`` under ``cascade.call_region``: equal call records and identical VCF rows.
``lstm_mufu16`` changes the gate math by design and is not compared across its settings.
"""
import threading

import numpy as np
import pytest
import torch

from clair3_b200 import bam_io, cascade, decode, sharding, synth, synth_reads as sr
from clair3_b200.model import Clair3_F, Clair3_P

pytestmark = pytest.mark.gpu

N_SITES = 2600                     # > 2 default pileup chunks, > 10 full-alignment chunks; ~2,300+ sites per chunk is where
                                   # a tile-and-SM-count split rule departed from the default-chunk split
FA_DEPTH = 55
SPECIAL = np.array([2047, 2048, 2049, 65504, 65519, 65520, 67552, 67553, 131008, 131009, 200000, 1000000])
SPECIAL = np.concatenate([SPECIAL, -SPECIAL])          # the hi / lo fp16 split's edges and counts far beyond any depth


def _same(got, want, what):
    """Bitwise equality of two float32 output blocks; on failure, how many rows differ, the largest |dp| and ulp distance."""
    got, want = torch.as_tensor(got).cpu(), torch.as_tensor(want).cpu()
    assert got.shape == want.shape, (what, tuple(got.shape), tuple(want.shape))
    if torch.equal(got, want):
        return
    g, w = got.numpy(), want.numpy()
    d = np.abs(g.astype(np.float64) - w)
    ulp = np.abs(g.view(np.int32).astype(np.int64) - w.view(np.int32).astype(np.int64))    # outputs are probabilities >= 0
    bad = int((d.max(1) > 0).sum()) if d.ndim == 2 else int((d > 0).sum())
    pytest.fail("%s: %d of %d rows differ, max |dp| %.3e, max %d ulp" % (what, bad, len(g), d.max(), ulp.max()))


def _model(cls, sd, channels, add_indel, **opts):
    m = cls(add_indel_length=add_indel, predict=True, input_channels=channels)
    m.set_option("precision", 0)
    for k, v in opts.items():
        m.set_option(k, v)
    m.to(torch.device("cuda"))
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    return m


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _into(m, xd, stream=None):
    y = torch.empty((xd.shape[0], m.out_dim), dtype=torch.float32, device="cuda")
    with torch.cuda.stream(stream or torch.cuda.current_stream()):
        m.forward_into(xd, y)
    return y


def _pileup_sites(n, seed):
    """Realistic per-strand counts with about 3 % of entries replaced by the special counts, and site 0 made of nothing but
    special counts; int32, exact in float32 too."""
    x = synth.pileup_inputs(n, seed=seed).astype(np.int64)
    r = np.random.default_rng(seed)
    mask = r.random(x.shape) < 0.03
    x[mask] = r.choice(SPECIAL, size=int(mask.sum()))
    x[0] = np.resize(SPECIAL, x.shape[1:])
    return x.astype(np.int32)


class Case:
    def __init__(self, cls, sd, channels, add_indel, x):
        self.cls, self.sd, self.channels, self.add, self.x = cls, sd, channels, add_indel, x
        self.m = _model(cls, sd, channels, add_indel)
        self.xd = _dev(x)
        self.want = self.m(self.xd)                    # the reference call: device tensors, default chunking
        torch.cuda.synchronize()

    def model(self, **opts):
        return _model(self.cls, self.sd, self.channels, self.add, **opts)

    def rows(self, idx):
        return self.want[torch.from_numpy(np.asarray(idx, dtype=np.int64)).cuda()]


@pytest.fixture(scope="module", params=[False, True], ids=["pileup24", "pileup90"])
def plp(request):
    add = request.param
    c = Case(Clair3_P, synth.pileup_state_dict(add, seed=81 + add), 18, add, _pileup_sites(N_SITES, 81))
    yield c
    c.m._release()


@pytest.fixture(scope="module", params=[8, 9], ids=["fa8", "fa9"])
def fa(request):
    ch = request.param
    c = Case(Clair3_F, synth.fa_state_dict(True, channels=ch, seed=82), ch, True,
             synth.fa_inputs(N_SITES, depth=FA_DEPTH, channels=ch, seed=82))
    yield c
    c.m._release()


# ---------------------------------------------------------------------------------------------- both networks
def _neighbours(c, m, sizes, seed):
    rng = np.random.default_rng(seed)
    for n in sizes:
        idx = rng.integers(0, N_SITES, size=n)                      # repeats, any order
        _same(m(_dev(c.x[idx])), c.rows(idx), "gathered %d" % n)
        lo = int(rng.integers(0, N_SITES - n + 1))                   # a contiguous run at another position
        _same(m(c.xd[lo:lo + n]), c.want[lo:lo + n], "slice %d at %d" % (n, lo))
    perm = rng.permutation(N_SITES)
    _same(m(_dev(c.x[perm])), c.rows(perm), "permutation")


def test_pileup_neighbours_and_position(plp):
    sizes = (1, 2, 127, 128, 129, 511, 512, 1023, 1024, 1025, 2200)
    _neighbours(plp, plp.m, sizes, 1)
    m = plp.model(chunk_sites=4096)                # every size in one chunk: the heads' 16-site groups and, at 2200 sites
    try:                                           # with add_indel, one block walking all head pairs
        _neighbours(plp, m, sizes, 2)
    finally:
        m._release()


def test_full_alignment_neighbours_and_position(fa):
    _neighbours(fa, fa.m, (1, 2, 3, 129, 255, 256, 257, 300), 3)


def _chunking(c, chunks):
    for chunk in chunks:
        m = c.model(chunk_sites=chunk)
        try:
            _same(m(c.xd), c.want, "chunk_sites %d" % chunk)
        finally:
            m._release()


def test_pileup_chunking(plp):
    _chunking(plp, (1, 7, 16, 128, 1000, 1024, 2304, 2600, 4096, 8192))


def test_full_alignment_chunking(fa):
    _chunking(fa, (1, 16, 100, 256, 1000, 4096))


def _call_shapes(c):
    m, x, want = c.m, c.x, c.want
    y = m(torch.from_numpy(x))                                       # host in, host out: latency mode
    assert y.device.type == "cpu"
    _same(y, want, "host forward")
    _same(_into(m, c.xd), want, "forward_into")

    cuts = (0, 700, 1500, N_SITES)
    streams = [torch.cuda.Stream() for _ in range(3)]
    xs = [torch.from_numpy(x[a:b]).pin_memory() for a, b in zip(cuts, cuts[1:])]
    ys = [torch.full((len(t), m.out_dim), -1.0).pin_memory() for t in xs]
    torch.cuda.synchronize()
    for rep in range(2):
        for s, xi, yi in zip(streams, xs, ys):
            with torch.cuda.stream(s):
                m.forward_async(xi, yi)
        torch.cuda.synchronize()
        _same(torch.cat(ys), want, "forward_async, repeat %d" % rep)

    sizes = (1, 300, 1024, 1100, 175)
    assert sum(sizes) == N_SITES
    parts = np.split(x, np.cumsum(sizes)[:-1])
    _same(torch.from_numpy(np.concatenate(list(m.predict_stream(iter(parts), streams=3)))), want, "predict_stream")

    rng = np.random.default_rng(4)
    idx = [rng.permutation(N_SITES)[:1100 + 100 * i] for i in range(8)]
    xd = [_dev(x[i]) for i in idx]
    streams = [torch.cuda.Stream() for _ in range(8)]
    torch.cuda.synchronize()
    for rep in range(3):
        outs = []
        for s, xi in zip(streams, xd):
            with torch.cuda.stream(s):
                outs.append(m(xi))
        torch.cuda.synchronize()
        for i, (o, ii) in enumerate(zip(outs, idx)):
            _same(o, c.rows(ii), "stream %d, repeat %d" % (i, rep))


def test_pileup_call_shapes(plp):
    _call_shapes(plp)


def test_full_alignment_call_shapes(fa):
    _call_shapes(fa)


def _two_threads(c):
    other = c.model()
    halves = ((0, 1300), (1300, N_SITES))
    results, errors = {}, []

    def run(k, m, lo, hi):
        try:
            s = torch.cuda.Stream()
            xd = c.xd[lo:hi]
            torch.cuda.current_stream().synchronize()
            for rep in range(3):
                y = _into(m, xd, s)
                s.synchronize()
                results[(k, rep)] = y
        except Exception as e:                     # reported by the main thread
            errors.append(e)

    try:
        threads = [threading.Thread(target=run, args=(k, m, lo, hi)) for k, (m, (lo, hi)) in enumerate(zip((c.m, other), halves))]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        assert not errors, errors
        for (k, rep), y in sorted(results.items()):
            lo, hi = halves[k]
            _same(y, c.want[lo:hi], "thread %d, repeat %d" % (k, rep))
        assert len(results) == 6
    finally:
        other._release()


def test_pileup_two_models_on_two_host_threads(plp):
    _two_threads(plp)


def test_full_alignment_two_models_on_two_host_threads(fa):
    _two_threads(fa)


def test_pileup_kernel_variants(plp):
    for tile in (16, 32, 64):
        for wg in (1, 2):
            m = plp.model(lstm_tile=tile, lstm_wg=wg)
            try:
                _same(m(plp.xd), plp.want, "lstm_tile %d, lstm_wg %d" % (tile, wg))
            finally:
                m._release()


def test_pileup_input_dtypes(plp):
    _same(plp.m(_dev(plp.x.astype(np.float32))), plp.want, "float32")
    x8 = synth.pileup_inputs(1100, seed=83, dtype=np.int8)
    y8 = plp.m(_dev(x8))
    for dt in (np.int32, np.float32):
        _same(plp.m(_dev(x8.astype(dt))), y8, np.dtype(dt).name)


def test_full_alignment_input_dtypes(fa):
    for dt in (np.int32, np.float32):
        _same(fa.m(_dev(fa.x.astype(dt))), fa.want, np.dtype(dt).name)


def _gather(cols, starts, bounds=None):
    """Host windows of forward_windows: rows starts[b] .. +32, zero outside the matrix and outside [bounds[b, 0], bounds[b, 1])."""
    rows = starts[:, None] + np.arange(33)[None, :]
    ok = (rows >= 0) & (rows < len(cols))
    if bounds is not None:
        ok &= (rows >= bounds[:, :1]) & (rows < bounds[:, 1:])
    out = np.zeros((len(starts), 33, cols.shape[1]), dtype=np.int64)
    out[ok] = cols[rows[ok]]
    return out.astype(np.int32)


def test_pileup_windows(plp):
    n_cols = 3000
    cols = _pileup_sites(-(-n_cols // 33), 84).reshape(-1, 18)[:n_cols].astype(np.int64)
    rng = np.random.default_rng(84)
    starts = rng.integers(-40, n_cols + 8, size=1100).astype(np.int64)       # overhanging both ends
    lo = starts + rng.integers(-5, 20, size=starts.shape)
    bounds = np.stack([lo, lo + rng.integers(0, 40, size=starts.shape)], axis=1).astype(np.int64)
    for bnd in (None, bounds):
        want = plp.m(_dev(_gather(cols, starts, bnd)))
        for dt in (np.int32, np.int64):
            got = plp.m.forward_windows(_dev(cols.astype(dt)), _dev(starts), bounds=None if bnd is None else _dev(bnd))
            _same(got, want, "windows %s, bounds %s" % (np.dtype(dt).name, bnd is not None))
        got = plp.m.forward_windows(torch.from_numpy(cols), torch.from_numpy(starts),
                                    bounds=None if bnd is None else torch.from_numpy(bnd))
        _same(got, want, "host windows int64, bounds %s" % (bnd is not None))


def _sharding(c):
    for world in (2, 3, 5, 8):
        parts = [c.m(c.xd[slice(*sharding.site_range(N_SITES, r, world))]) for r in range(world)]
        _same(torch.cat(parts), c.want, "world %d" % world)


def test_pileup_sharding(plp):
    _sharding(plp)


def test_full_alignment_sharding(fa):
    _sharding(fa)


def _repeatability(c):
    ys = [c.m(c.xd) for _ in range(3)]
    for i, y in enumerate(ys):
        _same(y, ys[0], "repeat %d" % i)
    _same(ys[0], c.want, "against the first call")


def test_pileup_repeatability(plp):
    _repeatability(plp)


def test_full_alignment_repeatability(fa):
    _repeatability(fa)


# ---------------------------------------------------------------------------------------------- one network
def test_l4_split_count_depends_on_k_only():
    """L4's grid is (tiles, splits) with the split count from K alone: 15 for the pileup net (165 k-chunks), 14 for full
    alignment (56), for one tile and for 21 tiles in one chunk alike."""
    from clair3_b200._ffi import check, ffi, lib
    cases = ((Clair3_P, synth.pileup_state_dict(True, seed=85), 18, lambda n: _pileup_sites(n, 85), 15),
             (Clair3_F, synth.fa_state_dict(True, channels=8, seed=85), 8,
              lambda n: synth.fa_inputs(n, depth=FA_DEPTH, channels=8, seed=85), 14))
    for cls, sd, ch, make, nsplit in cases:
        m = _model(cls, sd, ch, True, chunk_sites=4096)
        try:
            for n in (1, 129, 1024, N_SITES):
                xd = _dev(make(n))
                m.set_option("profile", 1)
                m(xd)
                torch.cuda.synchronize()
                ctas = ffi.new("double *")
                check(lib().c3b_get_profile_ctas(m._handle, b"tail", ctas))
                assert ctas[0] == nsplit * -(-n // 128), (cls.__name__, n, ctas[0])
        finally:
            m._release()


def test_pileup_64bit_offsets():
    """51 200 sites in one chunk: LSTM2's pre-gates are 33 x 51 200 x 1 280 > 2^31 fp16 elements (4.3 GB), so a 32-bit offset
    in proj2's stores or LSTM2's loads lands on another site's row.  About 7 GB of workspace, released at the end."""
    n = 51200
    sd = synth.pileup_state_dict(True, seed=86)
    x = _dev(_pileup_sites(n, 86))
    small = _model(Clair3_P, sd, 18, True)
    big = _model(Clair3_P, sd, 18, True, chunk_sites=n)
    try:
        want = small(x)
        _same(big(x), want, "one %d-site chunk" % n)
    finally:
        small._release()
        big._release()
        del x
        torch.cuda.empty_cache()


def test_full_alignment_workspace_history():
    """One model's calls in this order, each against a fresh model's output for the same call: 256 sites at depth 89 (the
    planar layout of a 256-site chunk), 3 at 89 (reuses it), 300 at 55 (a depth change), 44 at 55, 256 at 89 again.  The
    planar maps' zero borders must be cleared whenever the layout under them changes."""
    sd = synth.fa_state_dict(True, channels=8, seed=87)
    m = _model(Clair3_F, sd, 8, True)
    try:
        for n, depth in ((256, 89), (3, 89), (300, 55), (44, 55), (256, 89)):
            x = _dev(synth.fa_inputs(n, depth=depth, channels=8, seed=n + depth))
            got = m(x)
            fresh = _model(Clair3_F, sd, 8, True)
            try:
                _same(got, fresh(x), "%d sites at depth %d" % (n, depth))
            finally:
                fresh._release()
    finally:
        m._release()


# ---------------------------------------------------------------------------------------------- end to end
@pytest.fixture(scope="module")
def region(tmp_path_factory):
    """A 12 kb region at depth 24 with 2 kb reads, written as an indexed BAM."""
    rec, ref, rs = sr.random_alignment(12000, depth=24, read_len=2000, seed=61, origin=3000)
    path = str(tmp_path_factory.mktemp("tc_invariance") / "r.bam")
    bam_io.write_bam(path, rec, [("ctg", rs + len(ref))])
    bam_io.write_bai(path)
    return path, ref, rs, 3000, 15000


def test_call_region_independent_of_chunk_sites(region):
    path, ref, rs, start, end = region
    cfg_p = decode.replay_config(pileup=True, add_indel_length=False)._replace(is_show_reference=True)
    cfg_f = decode.replay_config(pileup=False, add_indel_length=True)._replace(is_show_reference=True)
    sd_p, sd_f = synth.pileup_state_dict(False, seed=1), synth.fa_state_dict(True, channels=8, seed=1)
    ws = cascade.Workspaces(0)
    runs = []
    try:
        for chunk in (0, 16, 4096):
            mp = _model(Clair3_P, sd_p, 18, False, chunk_sites=chunk)
            mf = _model(Clair3_F, sd_f, 8, True, chunk_sites=chunk)
            try:
                r = cascade.call_region(path, "ctg", start, end, ref, rs, mp, mf, cfg_p, cfg_f, print_ref=True, workspaces=ws)
                runs.append({"vcf": r["vcf"], "p": (r["pileup"]["Y"].clone(), r["pileup"]["device"]["calls"].clone()),
                             "f": [(f["Y"].clone(), f["device"]["calls"].clone()) for f in r["full_alignment"]]})
            finally:
                mp._release()
                mf._release()
    finally:
        ws.close()
    base = runs[0]
    assert len(base["p"][0]) > 0 and len(base["f"]) > 0 and base["vcf"]
    for chunk, r in zip((16, 4096), runs[1:]):
        _same(r["p"][0], base["p"][0], "pileup Y, chunk_sites %d" % chunk)
        assert torch.equal(r["p"][1], base["p"][1]), chunk
        assert len(r["f"]) == len(base["f"]), chunk
        for (y, calls), (y0, calls0) in zip(r["f"], base["f"]):
            _same(y, y0, "full-alignment Y, chunk_sites %d" % chunk)
            assert torch.equal(calls, calls0), chunk
        assert r["vcf"] == base["vcf"], chunk
