// inflate.cuh - RFC 1951 (DEFLATE) decoding of one BGZF block's payload and the CRC-32 of RFC 1952, for the BAM decoder
// (bam_decode.cu).  Everything here is __host__ __device__ and single-threaded, so the decoder's kernels and a host build share
// one statement of the format.  A malformed stream never makes the decoder read or write out of range: every input byte past
// the payload reads as zero and ends the block with INPUT_OVERRUN, every write is checked against the output capacity, and
// every back-reference against the bytes already produced.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define C3B_HD __host__ __device__ __forceinline__
#else
#define C3B_HD inline
#endif

namespace c3b_inflate {

// Status of one block (0 = inflated, CRC and size checked).  bam_decode.cu names them in its errors.
enum Status : int {
    OK = 0,
    BAD_BLOCK_TYPE = 1,     // BTYPE 11
    BAD_STORED_LENGTH,      // a stored block's NLEN is not the complement of LEN
    BAD_CODE_LENGTHS,       // a dynamic block's code lengths are malformed or over-subscribed
    BAD_CODE,               // a code that is not in the table, or a length / distance symbol outside the alphabet
    BAD_DISTANCE,           // a back-reference before the start of the block's output
    OUTPUT_OVERFLOW,        // more output than the block's ISIZE
    INPUT_OVERRUN,          // the stream reads past the block's compressed payload
    SIZE_MISMATCH,          // less output than ISIZE
    CRC_MISMATCH,
    N_STATUS
};

constexpr int FAST = 10;    // code bits one table lookup resolves; longer codes take the canonical bit-by-bit path

// A canonical Huffman code: the number of codes of each length, the symbols in code order, and the lookup table of the codes
// of at most FAST bits (entry = symbol << 4 | length, indexed by the next FAST stream bits; 0 = a longer code or none).
struct Huff {
    int16_t count[16];
    int16_t symbol[288];
    uint16_t fast[1 << FAST];
};
struct Tables {
    Huff lit, dist;
    uint8_t lengths[320];
};

// LSB-first bit reader over n bytes; bytes past the end read as zero and set `over`.
struct Bits {
    const uint8_t *in;
    int n, pos;
    int cnt;
    uint64_t buf;
    bool over;
    C3B_HD void need(int k) {
        while (cnt < k) {
            uint32_t b = 0;
            if (pos < n) {
#if defined(__CUDA_ARCH__)
                b = __ldg(in + pos);
#else
                b = in[pos];
#endif
            } else {
                over = true;
            }
            ++pos;
            buf |= (uint64_t)b << cnt;
            cnt += 8;
        }
    }
    C3B_HD void drop(int k) { buf >>= k; cnt -= k; }
    C3B_HD uint32_t bits(int k) {       // k <= 32
        if (k == 0) return 0;
        need(k);
        const uint32_t v = (uint32_t)(buf & ((1ull << k) - 1));
        drop(k);
        return v;
    }
    // Bytes read past the payload: the zeros that `need` supplied beyond n, less those still unread in the buffer.
    C3B_HD bool overran() const { return over && (int64_t)pos * 8 - cnt > (int64_t)n * 8; }
};

// Builds h from the code lengths of n symbols.  Returns false for an over-subscribed code; an incomplete one is accepted, and
// decoding one of its unassigned codes fails.
C3B_HD bool build(Huff &h, const uint8_t *len, int n) {
    for (int l = 0; l < 16; ++l) h.count[l] = 0;
    for (int s = 0; s < n; ++s) h.count[len[s]]++;
    int left = 1;
    for (int l = 1; l < 16; ++l) {
        left = (left << 1) - h.count[l];
        if (left < 0) return false;
    }
    int16_t offs[16];
    offs[1] = 0;
    for (int l = 1; l < 15; ++l) offs[l + 1] = offs[l] + h.count[l];
    for (int s = 0; s < n; ++s)
        if (len[s]) h.symbol[offs[len[s]]++] = (int16_t)s;
    for (int i = 0; i < (1 << FAST); ++i) h.fast[i] = 0;
    int code = 0, idx = 0;
    for (int l = 1; l <= FAST; ++l) {
        for (int k = 0; k < h.count[l]; ++k, ++code) {
            int rev = 0;
            for (int b = 0; b < l; ++b) rev |= ((code >> b) & 1) << (l - 1 - b);
            const uint16_t e = (uint16_t)(h.symbol[idx++] << 4 | l);
            for (int f = rev; f < (1 << FAST); f += 1 << l) h.fast[f] = e;
        }
        code <<= 1;
    }
    return true;
}

// The next symbol of code h, or -1 for a code the table does not hold.
C3B_HD int decode(Bits &b, const Huff &h) {
    b.need(15);
    const uint16_t e = h.fast[b.buf & ((1u << FAST) - 1)];
    if (e) {
        b.drop(e & 15);
        return e >> 4;
    }
    int code = 0, first = 0, index = 0;
    for (int l = 1; l < 16; ++l) {
        code |= (int)(b.buf >> (l - 1)) & 1;
        const int count = h.count[l];
        if (code - count < first) {
            b.drop(l);
            return h.symbol[index + (code - first)];
        }
        index += count;
        first = (first + count) << 1;
        code <<= 1;
    }
    return -1;
}

// Inflates the raw DEFLATE stream in[0 .. n_in) into out[0 .. cap).  *n_out: the bytes written.
C3B_HD int inflate(const uint8_t *in, int n_in, uint8_t *out, int cap, int *n_out, Tables &t) {
    Bits b{in, n_in, 0, 0, 0, false};
    int o = 0, last = 0;
    *n_out = 0;
    do {
        last = (int)b.bits(1);
        const int type = (int)b.bits(2);
        if (type == 0) {
            b.drop(b.cnt & 7);
            const uint32_t len = b.bits(16), nlen = b.bits(16);
            if (b.overran()) return INPUT_OVERRUN;
            if (len != (~nlen & 0xffffu)) return BAD_STORED_LENGTH;
            if (o + (int)len > cap) return OUTPUT_OVERFLOW;
            for (uint32_t i = 0; i < len; ++i) out[o++] = (uint8_t)b.bits(8);
            if (b.overran()) return INPUT_OVERRUN;
            continue;
        }
        if (type == 3) return BAD_BLOCK_TYPE;
        uint8_t *L = t.lengths;
        int nlen = 288, ndist = 30;
        if (type == 1) {
            for (int s = 0; s < 288; ++s) L[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
            for (int s = 0; s < 30; ++s) L[288 + s] = 5;
            if (!build(t.lit, L, 288) || !build(t.dist, L + 288, 30)) return BAD_CODE_LENGTHS;
        } else {
            nlen = (int)b.bits(5) + 257;
            ndist = (int)b.bits(5) + 1;
            const int ncode = (int)b.bits(4) + 4;
            if (nlen > 286 || ndist > 30) return BAD_CODE_LENGTHS;
            const char *order = "\x10\x11\x12\x00\x08\x07\x09\x06\x0a\x05\x0b\x04\x0c\x03\x0d\x02\x0e\x01\x0f";
            for (int i = 0; i < 19; ++i) L[(int)order[i]] = i < ncode ? (uint8_t)b.bits(3) : 0;
            if (!build(t.lit, L, 19)) return BAD_CODE_LENGTHS;
            int idx = 0;
            while (idx < nlen + ndist) {
                const int sym = decode(b, t.lit);
                if (b.overran()) return INPUT_OVERRUN;
                if (sym < 0) return BAD_CODE_LENGTHS;
                if (sym < 16) {
                    L[idx++] = (uint8_t)sym;
                    continue;
                }
                uint8_t v = 0;
                int rep;
                if (sym == 16) {
                    if (idx == 0) return BAD_CODE_LENGTHS;
                    v = L[idx - 1];
                    rep = 3 + (int)b.bits(2);
                } else if (sym == 17) {
                    rep = 3 + (int)b.bits(3);
                } else {
                    rep = 11 + (int)b.bits(7);
                }
                if (idx + rep > nlen + ndist) return BAD_CODE_LENGTHS;
                while (rep--) L[idx++] = v;
            }
            if (L[256] == 0) return BAD_CODE_LENGTHS;
            if (!build(t.lit, L, nlen) || !build(t.dist, L + nlen, ndist)) return BAD_CODE_LENGTHS;
        }
        for (;;) {
            if (b.overran()) return INPUT_OVERRUN;
            int sym = decode(b, t.lit);
            if (sym < 0) return BAD_CODE;
            if (sym < 256) {
                if (o >= cap) return OUTPUT_OVERFLOW;
                out[o++] = (uint8_t)sym;
                continue;
            }
            if (sym == 256) break;
            sym -= 257;
            if (sym >= 29) return BAD_CODE;
            // length 3..258: codes 257..264 carry no extra bits, then four codes per extra bit, and 285 is 258
            int len;
            if (sym < 8) len = 3 + sym;
            else if (sym == 28) len = 258;
            else {
                const int ext = (sym - 4) >> 2;
                len = ((4 + (sym & 3)) << ext) + 3 + (int)b.bits(ext);
            }
            const int ds = decode(b, t.dist);
            if (ds < 0 || ds >= 30) return BAD_CODE;
            // distance 1..32768: codes 0..3 carry no extra bits, then two codes per extra bit
            int dist;
            if (ds < 4) dist = ds + 1;
            else {
                const int ext = (ds >> 1) - 1;
                dist = ((2 + (ds & 1)) << ext) + 1 + (int)b.bits(ext);
            }
            if (dist > o) return BAD_DISTANCE;
            if (o + len > cap) return OUTPUT_OVERFLOW;
            // byte by byte: a distance shorter than the length reads what this copy wrote
            for (int i = 0; i < len; ++i, ++o) out[o] = out[o - dist];
        }
    } while (!last);
    *n_out = o;
    return b.overran() ? INPUT_OVERRUN : OK;
}

// ---- CRC-32 (reflected, polynomial 0xEDB88320) ----
// The register update over bytes is affine: R(s, A B) = shift(R(s, A), |B|) ^ R(0, B), where shift multiplies by x^(8 |B|)
// modulo the polynomial.  So a warp splits a block into 32 chunks, each lane computes R(0, chunk) and shifts it past the bytes
// that follow, and the XOR of the lanes' terms with shift(~0, n) is R(~0, block): the CRC before the final complement.
#define C3B_CRC_X2N {0x40000000u, 0x20000000u, 0x08000000u, 0x00800000u, 0x00008000u, 0xedb88320u, 0xb1e6b092u, 0xa06a2517u, \
                     0xed627daeu, 0x88d14467u, 0xd7bbfe6au, 0xec447f11u, 0x8e7ea170u, 0x6427800eu, 0x4d47bae0u, 0x09fe548fu, \
                     0x83852d0fu, 0x30362f1au, 0x7b5a9cc3u, 0x31fec169u, 0x9fec022au, 0x6c8dedc4u, 0x15d6874du, 0x5fde7a4eu, \
                     0xbad90e37u, 0x2e4e5eefu, 0x4eaba214u, 0xa8a472c0u, 0x429a969eu, 0x148d302au, 0xc40ba6d0u, 0xc4e22c3cu}
#if defined(__CUDACC__)
static __constant__ uint32_t crc_x2n_dev[32] = C3B_CRC_X2N;   // x^(2^k) modulo the polynomial
#endif
static const uint32_t crc_x2n_host[32] = C3B_CRC_X2N;

C3B_HD uint32_t crc_x2n(int k) {
#if defined(__CUDA_ARCH__)
    return crc_x2n_dev[k & 31];
#else
    return crc_x2n_host[k & 31];
#endif
}

// a * b modulo the polynomial (bit 31 = x^0)
C3B_HD uint32_t crc_mult(uint32_t a, uint32_t b) {
    uint32_t m = 1u << 31, p = 0;
    while (a) {
        if (a & m) {
            p ^= b;
            a &= ~m;
        }
        m >>= 1;
        b = b & 1 ? (b >> 1) ^ 0xedb88320u : b >> 1;
    }
    return p;
}

// s shifted past n zero bytes: s * x^(8 n)
C3B_HD uint32_t crc_shift(uint32_t s, uint32_t n) {
    uint32_t p = 1u << 31;
    for (int k = 3; n; n >>= 1, ++k)
        if (n & 1) p = crc_mult(crc_x2n(k), p);
    return crc_mult(p, s);
}

C3B_HD uint32_t crc_table_entry(uint32_t i) {
    for (int k = 0; k < 8; ++k) i = i & 1 ? (i >> 1) ^ 0xedb88320u : i >> 1;
    return i;
}

// R(s, p[0 .. n)) with the 256-entry byte table
C3B_HD uint32_t crc_update(const uint32_t *table, uint32_t s, const uint8_t *p, int n) {
    for (int i = 0; i < n; ++i) s = table[(s ^ p[i]) & 0xff] ^ (s >> 8);
    return s;
}

// The lane split of a warp's CRC-32 over p[0 .. n): lane l of 32 takes the chunk [l * c, min((l + 1) * c, n)), c = ceil(n / 32),
// and returns R(0, chunk) shifted past the bytes after it.  The CRC is crc_lanes_done(the XOR of the 32 terms, n).
C3B_HD uint32_t crc_lane_term(const uint32_t *table, const uint8_t *p, int n, int lane) {
    const int chunk = (n + 31) / 32, a = lane * chunk, e = a + chunk < n ? a + chunk : n;
    return a < e ? crc_shift(crc_update(table, 0, p + a, e - a), (uint32_t)(n - e)) : 0;
}
C3B_HD uint32_t crc_lanes_done(uint32_t x, int n) { return ~(x ^ crc_shift(0xffffffffu, (uint32_t)n)); }

}  // namespace c3b_inflate
