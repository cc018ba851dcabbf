"""The BGZF writer's compressor (``clair3_b200/csrc/deflate.cuh``) built for the host with AddressSanitizer and UBSan, against
zlib: every payload of the corpus (``bgzf_corpus``) must come out as exactly the block ``bam_io._bgzf_block`` writes, which is
``zlib.compressobj(6, zlib.DEFLATED, -15)``'s stream in the BGZF frame.  The header is ``__host__ __device__``, so this is the
same statement of zlib's rules the GPU's ``bgzf_deflate_kernel`` runs, and its CRC-32 comes from the same 32-lane split."""
import os
import struct
import sys
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import bgzf_corpus as bc  # noqa: E402
import deflate_craft as dc  # noqa: E402
from clair3_b200 import bam_io  # noqa: E402

pytestmark = pytest.mark.skipif(zlib.ZLIB_RUNTIME_VERSION != bc.ZLIB_VERSION,
                                reason="byte equality is held to zlib %s; this Python links zlib %s"
                                % (bc.ZLIB_VERSION, zlib.ZLIB_RUNTIME_VERSION))


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    exe = bc.build_host_deflater(str(tmp_path_factory.mktemp("deflate_host")))
    if exe is None:
        pytest.skip("needs g++ for the sanitized host build")
    return exe


def _cases(payloads):
    return b"".join(struct.pack("<I", len(p)) + p for p in payloads)


def run_blocks(exe, payloads, mode="bgzf"):
    out = dc.run_host(exe, mode, _cases(payloads))
    res, o = [], 0
    for _ in payloads:
        n, = struct.unpack_from("<i", out, o)
        o += 4
        res.append(out[o:o + max(n, 0)] if n >= 0 else None)
        o += max(n, 0)
    assert o == len(out)
    return res


def run_parallel(exe, jobs, mode="bgzf"):
    """run_blocks over each payload list of ``jobs``, one driver process per list, as many at once as there are CPUs."""
    with ThreadPoolExecutor(max_workers=max(1, min(len(jobs), os.cpu_count() or 1))) as ex:
        return list(ex.map(lambda ps: run_blocks(exe, ps, mode), jobs))


def test_corpus_has_its_features(driver):
    """Each rule the corpus exists for runs somewhere in it: stored, fixed and dynamic blocks, a payload that flushes the
    symbol buffer several times, gen_bitlen's overflow repair, and the window slide."""
    cases = bc.payloads(0, mixtures=300)
    seen = np.frombuffer(dc.run_host(driver, "seen", _cases([p for _, p in cases])), dtype="<i4").reshape(-1, 5)
    named = dict(zip((n for n, _ in cases), seen))
    assert named["random, 0xFF00 bytes"][0] >= 4                        # stored, one per flush of the symbol buffer
    assert named["empty"][1] == 1 and named["1 byte"][1] == 1             # fixed
    assert named["symbol buffer flushes several times"][2] >= 2          # dynamic, flushed on the symbol buffer
    assert named["one byte, 0xFF00"][4] == 1 and named["text, 0xFF00 - 1 bytes"][4] == 1 and named["random, 1000"][4] == 0
    assert (seen[:, 3] > 0).sum() >= 20                                   # overflow repairs
    assert (seen[:, 0] > 0).sum() and (seen[:, 1] > 0).sum() and (seen[:, 2] > 0).sum()


def test_blocks_equal_zlibs(driver):
    """The named cases and 3,000 seeded mixtures, block for block."""
    cases = bc.payloads(1, mixtures=3000)
    ps = [p for _, p in cases]
    got = [g for gs in run_parallel(driver, [ps[i:i + 400] for i in range(0, len(ps), 400)]) for g in gs]
    for (name, p), g in zip(cases, got):
        assert g == bam_io._bgzf_block(p), (name, len(p))


def _cta_jobs(cases, k, seed):
    """The payload sequences the ``cta k`` runs take: the cases in three seeded orders, then every case on a state that has
    just compressed a full-size random block and one that has just compressed a full-size run block (per group of k cases:
    k random blocks, the k cases, k run blocks, the k cases again, so case j of the group lands on state j after each).  The
    second part is cut into several runs (every run starts on fresh, poisoned states) so that they can go in parallel."""
    rng = np.random.default_rng(seed)
    rnd = rng.integers(0, 256, bc.PAYLOAD, dtype=np.uint8).tobytes()
    run = b"".join(bytes([65 + i]) * (bc.PAYLOAD // 4) for i in range(4))
    jobs = [[cases[i] for i in rng.permutation(len(cases))] for _ in range(3)]
    after = []
    for g in range(0, len(cases), k):
        grp = cases[g:g + k]
        after += [rnd] * len(grp) + grp + [run] * len(grp) + grp
    step = -(-len(after) // (4 * 4 * k)) * 4 * k       # whole groups per run
    return jobs + [after[i:i + step] for i in range(0, len(after), step)], (rnd, run)


@pytest.mark.parametrize("k", [1, 3])
def test_blocks_equal_zlibs_on_reused_state(driver, k):
    """The kernel's CTA c compresses blocks c, c + grid, ... on one state: its window, head, prev, trees and symbol buffer keep
    whatever the block before left there, and only reset_block runs between.  ``cta k`` holds k such states, every byte
    poisoned first, and sends payload i to state i % k: each block must still be exactly zlib's.  The named cases and 1,500
    mixtures in three orders, and each of them right after a full-size random block and a full-size run block."""
    cases = [p for _, p in bc.payloads(5, mixtures=1500)]
    jobs, full = _cta_jobs(cases, k, 17 + k)
    want = {p: bam_io._bgzf_block(p) for p in cases + list(full)}
    got = run_parallel(driver, jobs, "cta %d" % k)
    for ps, gs in zip(jobs, got):
        for i, (p, g) in enumerate(zip(ps, gs)):
            assert g == want[p], (k, i, len(p))


def test_vcf_texts_equal_the_host_writer(driver, tmp_path):
    """Whole files: VCF-like texts of many blocks, cut into 0xFF00-byte blocks and framed with the EOF block, equal
    bam_io.write_bgzf's file.  (The genome route's own files are compared on the GPU, in test_gpu_bgzf_write.py.)"""
    for _, t in bc.texts(3):
        blocks = run_blocks(driver, [t[i:i + bc.PAYLOAD] for i in range(0, len(t), bc.PAYLOAD)])
        path = str(tmp_path / "host.gz")
        bam_io.write_bgzf(path, t)
        with open(path, "rb") as f:
            assert b"".join(blocks) + bam_io._EOF == f.read()
