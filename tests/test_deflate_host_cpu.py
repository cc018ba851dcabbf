"""The BGZF writer's compressor (``clair3_b200/csrc/deflate.cuh``) built for the host with AddressSanitizer and UBSan, against
zlib: every payload of the corpus (``bgzf_corpus``) must come out as exactly the block ``bam_io._bgzf_block`` writes, which is
``zlib.compressobj(6, zlib.DEFLATED, -15)``'s stream in the BGZF frame.  The header is ``__host__ __device__``, so this is the
same statement of zlib's rules the GPU's ``bgzf_deflate_kernel`` runs, and its CRC-32 comes from the same 32-lane split."""
import os
import struct
import sys
import zlib

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


def run_blocks(exe, payloads):
    out = dc.run_host(exe, "bgzf", _cases(payloads))
    res, o = [], 0
    for _ in payloads:
        n, = struct.unpack_from("<i", out, o)
        o += 4
        res.append(out[o:o + max(n, 0)] if n >= 0 else None)
        o += max(n, 0)
    assert o == len(out)
    return res


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
    got = run_blocks(driver, [p for _, p in cases])
    for (name, p), g in zip(cases, got):
        assert g == bam_io._bgzf_block(p), (name, len(p))


def test_vcf_texts_equal_the_host_writer(driver, tmp_path):
    """Whole files: VCF-like texts of many blocks, cut into 0xFF00-byte blocks and framed with the EOF block, equal
    bam_io.write_bgzf's file.  (The genome route's own files are compared on the GPU, in test_gpu_bgzf_write.py.)"""
    for _, t in bc.texts(3):
        blocks = run_blocks(driver, [t[i:i + bc.PAYLOAD] for i in range(0, len(t), bc.PAYLOAD)])
        path = str(tmp_path / "host.gz")
        bam_io.write_bgzf(path, t)
        with open(path, "rb") as f:
            assert b"".join(blocks) + bam_io._EOF == f.read()
