"""Mints tests/golden/fa_ref_cases.npz from the reference's own calculate_clair3_full_alignment, compiled by oracle/fa_ref.py (needs
the reference checkout: CLAIR3_REFERENCE or a sibling directory).

For every targeted case of tests/fa_ref_cases.py (the inputs are rebuilt from that module's code) it stores the reference's
matrix, its all_alt_info strings and the number of rand() draws it consumed, under ``<name>/matrix``, ``<name>/alt_info`` and
``<name>/draws``, so that those cases pin the GPU builder even where oracle/_ref/ was not built.  At every large ``rand_skip`` it
also checks ``clair3_b200.fa_tensor.glibc_rand`` (the jump-ahead restatement the GPU builder shares) against the C library's own
rand() stepped that far, and stores the 80 values under ``glibc_rand/<skip>``.

The large-skip cases step glibc's rand() up to 2^32 + 12345 times in a C loop; on a 2020s x86-64 core that is about 17 ns a draw,
so the script takes about four minutes.
    python tests/golden/make_fa_ref_cases_golden.py"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from clair3_b200.fa_tensor import glibc_rand  # noqa: E402
from oracle import fa_ref  # noqa: E402
import fa_ref_cases as cases  # noqa: E402

if fa_ref.build() is None:
    sys.exit("the reference checkout is needed: set CLAIR3_REFERENCE")

out = {"names": np.array([n for n, _ in cases.TARGETED])}
for skip in cases.LARGE_SKIPS:
    t = time.time()
    want = fa_ref.libc_rand(1, 80, skip=skip)
    got = glibc_rand(1, skip, 80)
    if not np.array_equal(got, want):
        sys.exit("glibc_rand(1, %d) differs from the C library's rand()" % skip)
    out["glibc_rand/%d" % skip] = want
    print("rand_skip %d: glibc_rand equals the C library (%.1f s)" % (skip, time.time() - t))
for name, build in cases.TARGETED:
    t = time.time()
    rec, ref, cand, var, p = build()
    m, alt, draws = fa_ref.full_alignment(rec, cand, ref, variants=var, **p)
    out["%s/matrix" % name] = m
    out["%s/alt_info" % name] = np.array(alt, dtype=str)
    out["%s/draws" % name] = np.int64(draws)
    if time.time() - t > 1:
        print("%s: %.1f s" % (name, time.time() - t))
path = os.path.join(ROOT, "tests", "golden", "fa_ref_cases.npz")
np.savez_compressed(path, **out)
print("%d targeted cases, %d bytes" % (len(cases.TARGETED), os.path.getsize(path)))
