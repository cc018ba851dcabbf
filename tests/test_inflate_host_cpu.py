"""The BAM reader's inflater (``clair3_b200/csrc/inflate.cuh``) built for the host with AddressSanitizer and UBSan, against zlib on
a corpus of crafted DEFLATE streams (``deflate_craft``): the features real BAM writers emit and zlib's compressor does not, and
malformed streams that must end with a named status.  The header is ``__host__ __device__``, so this is the same statement of
the format the GPU's ``bam_inflate_kernel`` runs; the CRC-32 pieces its warp uses are checked here against ``zlib.crc32``."""
import os
import struct
import sys
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import deflate_craft as dc  # noqa: E402


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    exe = dc.build_host_inflater(str(tmp_path_factory.mktemp("inflate_host")))
    if exe is None:
        pytest.skip("needs g++ for the sanitized host build")
    return exe


def test_corpus_has_its_features():
    """The features the corpus exists for are really in it, so it cannot go stale silently."""
    c = dict(dc.corpus())

    def dyn(name):
        return [(b, *dc.block_lengths(b)) for b in c[name] if b["kind"] == "dynamic"]

    (b, L, D), = dyn("run crosses into distances")
    assert dc.dynamic_header(L, D, joint=True)[2] and not dc.dynamic_header(L, D, joint=False)[2]
    (b, L, D), = dyn("codes of 11-15 bits")
    lit_used, dist_used = dc._counts(b["syms"])
    assert {L[s] for s in range(286) if lit_used[s]} >= set(range(11, 16))
    assert {D[s] for s in range(30) if dist_used[s]} >= set(range(11, 16))
    (b, L, D), = dyn("one distance code")
    assert sorted(x for x in D if x) == [1]
    (b, L, D), = dyn("no distance code")
    assert not any(D)
    (b, L, D), = dyn("HLIT 257, 8 code-length codes")
    hb, _, _, nlit, _ = dc.dynamic_header(L, D)
    assert nlit == 257 and (hb.out[1] >> 2) & 15 == 4            # HLIT field 0 and HCLEN field 4 (8 code-length codes)
    kinds = [b["kind"] for b in c["stored, fixed, dynamic and empty stored blocks"]]
    assert {"stored", "fixed", "dynamic"} <= set(kinds)
    assert sum(1 for b in c["stored, fixed, dynamic and empty stored blocks"] if b["kind"] == "stored" and not b["data"]) >= 2
    far = [s for b in c["length 258 as 285 and 284+31, distance 32768, distance 1 and 2"] for s in b.get("syms", [])]
    assert dc.Match(258, 32768, 284) in far and dc.Match(258, 32768) in far
    assert any(isinstance(s, dc.Match) and s.dist == 1 for s in far) and any(isinstance(s, dc.Match) and s.dist == 2 for s in far)


def _valid_cases():
    cases = [(name, *dc.check(blocks)) for name, blocks in dc.corpus()]
    rng = np.random.default_rng(5)
    for mode in dc.MODES:
        for n in (1, 31, 32, 33, 4097, 40000):
            data = bytes(rng.integers(0, 7, n).astype(np.uint8) + 65)
            cases.append(("%s %d" % (mode, n), dc.encode_mode(data, mode, rng), data))
    return cases


def test_valid_streams_inflate_to_zlibs_bytes(driver):
    cases = _valid_cases()
    runs = [(s, len(want)) for _, s, want in cases] + [(s, len(want) + 77) for _, s, want in cases]
    got = dc.run_host_inflater(driver, runs)
    for (name, s, want), (st, out), (st2, out2) in zip(cases, got[:len(cases)], got[len(cases):]):
        assert zlib.decompress(s, -15) == want
        assert st == 0 and out == want, (name, st, len(out), len(want))
        assert st2 == 0 and out2 == want, (name, "larger capacity", st2)


def test_malformed_streams_end_with_their_status(driver):
    cases = dc.malformed()
    got = dc.run_host_inflater(driver, [(s, cap) for _, s, cap, _ in cases])
    for (name, _, _, status), (st, _) in zip(cases, got):
        assert st == dc.STATUS[status], (name, st, status)


def test_every_truncation_and_bit_flip_is_safe(driver):
    """Every prefix of a few streams, and single-bit flips, run under the sanitizers: any status, no report; a prefix that still
    inflates gives a prefix of the bytes."""
    base = [dc.check(blocks) for name, blocks in dc.corpus() if name in (
        "run crosses into distances", "codes of 11-15 bits", "stored, fixed, dynamic and empty stored blocks", "one distance code")]
    runs, want = [], []
    for s, data in base:
        for k in range(len(s)):
            runs.append((s[:k], len(data)))
            want.append(data)
        for k in range(0, 8 * len(s), 7):
            f = bytearray(s)
            f[k >> 3] ^= 1 << (k & 7)
            runs.append((bytes(f), len(data)))
            want.append(None)
    got = dc.run_host_inflater(driver, runs)
    for (s, _), w, (st, out) in zip(runs, want, got):
        assert 0 <= st < 8
        if st == 0 and w is not None:
            assert w.startswith(out)


def test_crc_pieces_match_zlib(driver):
    """crc_shift / crc_mult composition for every length 0..2048 (and a split point in each), and bam_inflate_kernel's 32-lane
    split for every residue of the length mod 32 and for 65,535 and 65,536 bytes."""
    rng = np.random.default_rng(9)
    buf = rng.integers(0, 256, 65536, dtype=np.uint8).tobytes()
    cases = [(n, int(rng.integers(0, n + 1))) for n in range(2049)]
    cases += [(32 * 37 + r, 5 * r) for r in range(32)] + [(65535, 65535), (65536, 0), (65536, 32768)]
    out = dc.run_host(driver, "crc", b"".join(struct.pack("<II", n, k) + buf[:n] for n, k in cases)).decode().split("\n")
    for (n, k), line in zip(cases, out):
        want = zlib.crc32(buf[:n]) & 0xFFFFFFFF
        assert [int(x, 16) for x in line.split()] == [want] * 3, (n, k, line)
