// alt_text.cuh - what the two all_alt_info text stages share: the pileup counter's (plp_alt_text.cu) and the full-alignment
// builder's (fa_alt_text.cu).  Both measure each candidate's string with a counting sink, scan the lengths, and write it again
// with a bounded sink; both order a kind of allele by replaying klib's khash (src/khash.h) over it.
#pragma once
#include <stdint.h>

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

}  // namespace
