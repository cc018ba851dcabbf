// alt_text.cuh - what the two all_alt_info text stages share: the pileup counter's (plp_alt_text.cu) and the full-alignment
// builder's (fa_alt_text.cu).  Candidates are independent and their strings have data-dependent length, so each stage is
//
//   measure   the stage's own kernel, one WARP per candidate: orders the candidate's allele records - each kind by replaying
//             klib's khash (src/khash.h) over it - then lane 0 walks the string once with a counting sink (text_measure_tail)
//   scan      two one-CTA exclusive scans (block_scan.cuh) over n_cand + 1 lengths: per-candidate offsets and the byte totals
//   write     text_write_kernel, one THREAD per candidate: walks the same string with a sink bounded by what measure found
//
// launched by text_launch.  A stage is a struct with its argument type (derived from C3bAltText), the candidate count as the
// kernels read it and as the scans take it, a candidate's position and the reference byte there, and emit: the walk over one
// candidate's string into a TextOut.  Same records, same bytes, whatever the launch shape: nothing is atomic but the status word.
#pragma once
#include <limits.h>
#include <stdint.h>

#include "block_scan.cuh"
#include "c3b_internal.h"

// Each translation unit keeps its own copies: the library is built without relocatable device code.
namespace {

__constant__ char NT16[17] = "=ACMGRSVTWYHKDBN";          // htslib seq_nt16_str

struct CountSink {
    long long n = 0;
    __device__ __forceinline__ void put(char) { ++n; }
};
struct WriteSink {              // writes inside [p, p + lim) only: lim is the length the measure pass found
    char *p;
    long long lim, n = 0;
    __device__ __forceinline__ void put(char c) { if (n < lim) p[n] = c; ++n; }
};

template <class S> struct TextOut {
    S full, dec;                // the reference's string, and "<depth>-<alt>" as the decoder takes it
    bool cut = false;           // the alt field of rstrip().split("-") ends at the first '-' of the alt text
    long long n_alt = 0;
    __device__ __forceinline__ void head(char c, bool both) {
        full.put(c);
        if (both) dec.put(c);
    }
    __device__ __forceinline__ void alt(char c) {
        full.put(c);
        ++n_alt;
        if (c == '-') cut = true;
        if (!cut) dec.put(c);
    }
    enum Where { HEAD_FULL, HEAD_BOTH, ALT };
    __device__ void num(long long v, Where w) {             // %d of a non-negative count, without a digit buffer
        unsigned long long u = (unsigned long long)v, p = 1;
        while (u / p >= 10) p *= 10;
        for (; p; p /= 10) {
            const char c = (char)('0' + (u / p) % 10);
            if (w == ALT) alt(c); else head(c, w == HEAD_BOTH);
        }
    }
};

// A khash bucket: key + 1 | old flag | new flag.  Keys are allele-record indices, below 2^24.
constexpr uint32_t KH_VAL = 0xffffffu, KH_OCC = 1u << 24, KH_TAKEN = 1u << 25;

// kh_resize (src/khash.h:246-306) for an insert-only table of n buckets; hash[key] is the key's hash.  Returns the new bucket
// count, 0 when the `avail` buckets at slot cannot hold it.
__device__ int khash_grow(const uint32_t *hash, uint32_t *slot, const int n, const int avail) {
    const int nn = n < 4 ? 4 : 2 * n;
    if (nn > avail) return 0;
    for (int b = 0; b < nn; ++b) {
        const uint32_t v = b < n ? (slot[b] & KH_VAL) : 0u;
        slot[b] = v | (v ? KH_OCC : 0u);
    }
    const uint32_t mask = (uint32_t)nn - 1u;
    for (int b = 0; b < n; ++b) {
        if (!(slot[b] & KH_OCC)) continue;
        uint32_t cur = slot[b] & KH_VAL;
        slot[b] &= KH_TAKEN;                                  // the bucket is free in the old table; its new flag stays
        for (;;) {                                            // kick-out: the evicted key is placed next
            uint32_t i = hash[cur - 1] & mask, step = 0;
            while (slot[i] & KH_TAKEN) i = (i + (++step)) & mask;
            const uint32_t e = slot[i];
            slot[i] = cur | KH_TAKEN;
            if (!(e & KH_OCC)) break;
            cur = e & KH_VAL;
        }
    }
    return nn;
}

// kh_put of the n distinct keys[0 .. n) in that order - power-of-two tables from 4, triangular probing, growth at 0.77 load at
// the start of a put - then, when `again` (a put of a present key followed the last new one), the growth that put still makes
// (khash.h:310-318).  Leaves keys[] in bucket order, the order kh_begin .. kh_end visits them.  False when the table would
// outgrow the `avail` buckets at slot; keys[] is then unchanged.
__device__ bool khash_replay(const uint32_t *hash, int32_t *keys, const int n, const bool again, uint32_t *slot, const int avail) {
    int nb = 0, size = 0, upper = 0;
    for (int k = 0; k < n; ++k) {
        if (size >= upper) {                                  // kh_put grows a full table before it looks the key up
            nb = khash_grow(hash, slot, nb, avail);
            if (!nb) return false;
            upper = (int)(nb * 0.77 + 0.5);
        }
        const uint32_t mask = (uint32_t)nb - 1u;
        uint32_t i = hash[keys[k]] & mask, step = 0;
        while (slot[i] & KH_VAL) i = (i + (++step)) & mask;
        slot[i] = (uint32_t)keys[k] + 1u;
        ++size;
    }
    if (n > 0 && again && size >= upper) {
        nb = khash_grow(hash, slot, nb, avail);
        if (!nb) return false;
    }
    int k = 0;
    for (int b = 0; b < nb; ++b)
        if (slot[b] & KH_VAL) keys[k++] = (int32_t)(slot[b] & KH_VAL) - 1;
    return true;
}

// Lane 0 of a measure kernel, once the stage has left candidate j's ni insertions and nd deletions in `order` (fits: its records
// and khash tables fitted the scratch): measures the string and stores what the scans, the write kernel and the decoder read.
template <class Stage>
__device__ void text_measure_tail(const typename Stage::Args &A, const int64_t j, bool fits, int ni, int nd) {
    if (!fits) { atomicOr(A.status, 1); ni = nd = 0; }
    A.n_ins[j] = ni;
    A.n_del[j] = nd;
    TextOut<CountSink> o;
    Stage::emit(A, j, ni, nd, o);
    if (!o.cut && o.n_alt > 0) --o.dec.n;                     // rstrip(): the alt text ends in one space
    if (!fits || o.full.n > INT_MAX || o.dec.n > INT_MAX) {
        atomicOr(A.status, 1);
        o.full.n = o.dec.n = 0;
    }
    A.len_text[j] = (int32_t)o.full.n;
    A.len_dec[j] = (int32_t)o.dec.n;
    const int64_t pos = Stage::pos(A, j);
    A.ref_base[j] = (uint8_t)Stage::ref_base(A, pos);
    A.position[j] = pos + 1;
}

template <class Stage> __global__ void __launch_bounds__(128) text_write_kernel(typename Stage::Args A) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= Stage::n_cand(A)) return;
    const int64_t t0 = A.text_off[j], t1 = A.text_off[j + 1], d0 = A.dec_off[j], d1 = A.dec_off[j + 1];
    if (t1 > A.text_cap || d1 > A.dec_cap) { atomicOr(A.status, 1); return; }
    TextOut<WriteSink> o;
    o.full.p = A.text + t0; o.full.lim = t1 - t0;
    o.dec.p = A.dec + d0; o.dec.lim = d1 - d0;
    if (t1 > t0) Stage::emit(A, j, A.n_ins[j], A.n_del[j], o);
}

// Queues a stage on stream s: measure, the two scans and text_write_kernel, sized from the bound a.n.  An empty stage writes the
// one offset of each scan instead.  `who` names the entry point in the errors.
template <class Stage>
int text_launch(const typename Stage::Args &a, void (*measure)(typename Stage::Args), cudaStream_t s, int *launches, const char *who) {
    if (a.n == 0) {
        C3B_CUDA(cudaMemsetAsync(a.text_off, 0, 8, s));
        C3B_CUDA(cudaMemsetAsync(a.dec_off, 0, 8, s));
        return 0;
    }
    if (a.al_cap >= (int64_t)KH_VAL) {
        c3b_set_error("%s: %lld allele records exceed the khash replay's 24-bit record index", who, (long long)a.al_cap);
        return 1;
    }
    int64_t blocks = ((a.n + 1) * 32 + 255) / 256;
    if (blocks > 132 * 8) blocks = 132 * 8;
    measure<<<(unsigned)blocks, 256, 0, s>>>(a);
    block_scan_sum(a.len_text, a.text_off, a.n + 1, Stage::n_cand_dev(a), a.totals, s);
    block_scan_sum(a.len_dec, a.dec_off, a.n + 1, Stage::n_cand_dev(a), a.totals + 1, s);
    text_write_kernel<Stage><<<(unsigned)((a.n + 127) / 128), 128, 0, s>>>(a);
    C3B_CUDA(cudaGetLastError());
    *launches = 4;
    return 0;
}

}  // namespace
