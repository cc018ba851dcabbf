// deflate.cuh - RFC 1951 (DEFLATE) compression of one BGZF block's payload, byte for byte as zlib 1.3 writes it at level 6
// (zlib.compressobj(6, zlib.DEFLATED, -15): windowBits 15, memLevel 8, the default strategy), for the BGZF writer in
// bam_decode.cu.  BGZF blocks are independent raw-deflate streams, so the GPU compresses one per CTA; everything here is
// __host__ __device__ and single-threaded, so the kernel and a host build (tests/deflate_host.cpp) share one statement.
//
// What is restated, and why each part matters to the bytes:
//   deflate.c  deflate_slow (lazy matching) with level 6's configuration (good 8, lazy 16, nice 128, chain 128), longest_match
//              with its stop rules (nice_match, the MAX_DIST limit, the chain cut to a quarter at prev_length >= good, the clamp
//              to the lookahead), the TOO_FAR drop of a far length-3 match, the rolling hash (15 bits, shift 5), head / prev,
//              and fill_window: its zeroing of the 258 bytes past the data and its slide at strstart >= w_size + MAX_DIST,
//              which a 65,280-byte payload reaches.  longest_match reads up to 258 bytes past strstart, past the data, and what
//              it finds there picks between matches of equal clamped length, so the window holds exactly zlib's bytes.
//   trees.c    _tr_tally into a symbol buffer that asks for a flush at lit_bufsize - 1 = 16,383 symbols; _tr_flush_block's
//              stored / fixed / dynamic choice; build_tree (the heap with its depth tie-break), gen_bitlen with its overflow
//              repair, gen_codes; build_bl_tree, scan_tree / send_tree; the bit buffer and bi_windup.
// Python's writer calls compress() and then flush(): deflate(Z_NO_FLUSH) stops at the first loop iteration whose lookahead is
// below MIN_LOOKAHEAD, and deflate(Z_FINISH) resumes there with a second fill_window that finds the same state (no input is
// left, and a slide the first call made leaves strstart below the slide point), so the stream is one Z_FINISH pass.
#pragma once
#include <stdint.h>

#include "inflate.cuh"

namespace c3b_deflate {

constexpr int W_SIZE = 32768, W_MASK = W_SIZE - 1, WINDOW = 2 * W_SIZE;
constexpr int HASH_SHIFT = 5, HASH_MASK = 32767;                 // hash_bits = memLevel 8 + 7
constexpr int MIN_MATCH = 3, MAX_MATCH = 258, MIN_LOOKAHEAD = MAX_MATCH + MIN_MATCH + 1, MAX_DIST = W_SIZE - MIN_LOOKAHEAD;
constexpr int TOO_FAR = 4096, WIN_INIT = MAX_MATCH;
constexpr unsigned GOOD = 8, LAZY = 16, NICE = 128, CHAIN = 128;   // configuration_table[6]
constexpr int SYM_END = (16384 - 1) * 3;                          // (lit_bufsize - 1) * 3 bytes of (dist, length / literal)
constexpr int L_CODES = 286, D_CODES = 30, BL_CODES = 19, HEAP_SIZE = 2 * L_CODES + 1, MAX_BITS = 15, MAX_BL_BITS = 7;
constexpr int END_BLOCK = 256, REP_3_6 = 16, REPZ_3_10 = 17, REPZ_11_138 = 18;

// BGZF framing, as clair3_b200/bam_io.py: _bgzf_block writes it
constexpr int PAYLOAD = 0xFF00, BLOCK_MAX = 65536, HEADER = 18, FOOTER = 8;
enum Status : int { OK = 0, OUTPUT_OVERFLOW = 1 };

// One Huffman tree (trees.c's ct_data with its unions split: freq / code and dad / len): leaves, then the internal nodes.
struct Tree {
    uint16_t *freq, *dad, *len, *code;
    int elems, extra_base, max_length, max_code;
    int kind;                           // 0 literal / length, 1 distance, 2 bit length: picks the extra bits
    const uint8_t *static_len;          // the static tree's lengths, or null (bit-length tree)
};

template <int N> struct TreeStore {
    uint16_t freq[N], dad[N], len[N + 1], code[N];
};

// Everything a block's Huffman stage keeps; the kernel holds it in shared memory.
struct Trees {
    TreeStore<HEAP_SIZE> l;
    TreeStore<2 * D_CODES + 1> d;
    TreeStore<2 * BL_CODES + 1> bl;
    uint16_t s_lcode[288], s_dcode[D_CODES];
    uint8_t s_llen[288], s_dlen[D_CODES];
    int16_t heap[HEAP_SIZE];
    uint8_t depth[HEAP_SIZE];
    uint16_t bl_count[MAX_BITS + 1];
    int heap_len, heap_max;
};

C3B_HD int lextra(int c) { return c < 8 || c == 28 ? 0 : (c - 4) >> 2; }
C3B_HD int dextra(int c) { return c < 4 ? 0 : (c >> 1) - 1; }
C3B_HD int blextra(int c) { return c == 16 ? 2 : c == 17 ? 3 : c == 18 ? 7 : 0; }
C3B_HD int log2i(unsigned v) {
    int k = 0;
    while (v >> (k + 1)) ++k;
    return k;
}
// _length_code[lc] for lc = length - 3 (0..255), and base_length
C3B_HD int length_code(unsigned lc) {
    if (lc < 8) return (int)lc;
    if (lc == 255) return 28;
    const int k = log2i(lc);
    return 4 * (k - 1) + (int)((lc >> (k - 2)) & 3);
}
C3B_HD unsigned base_length(int c) { return c < 8 ? (unsigned)c : (unsigned)(4 + (c & 3)) << ((c - 4) >> 2); }
// d_code(dist) for dist = distance - 1 (0..32767), and base_dist
C3B_HD int dist_code(unsigned d) {
    if (d < 4) return (int)d;
    const int k = log2i(d);
    return 2 * k + (int)((d >> (k - 1)) & 1);
}
C3B_HD unsigned base_dist(int c) { return c < 4 ? (unsigned)c : (unsigned)(2 + (c & 1)) << ((c >> 1) - 1); }

C3B_HD unsigned bi_reverse(unsigned code, int len) {
    unsigned r = 0;
    do {
        r |= code & 1;
        code >>= 1, r <<= 1;
    } while (--len > 0);
    return r >> 1;
}

// gen_codes: the canonical codes of tree[0 .. max_code] from their lengths and bl_count
template <class Len> C3B_HD void gen_codes(uint16_t *code, const Len *len, int max_code, const uint16_t *bl_count) {
    uint16_t next[MAX_BITS + 1];
    unsigned c = 0;
    for (int bits = 1; bits <= MAX_BITS; ++bits) {
        c = (c + bl_count[bits - 1]) << 1;
        next[bits] = (uint16_t)c;
    }
    for (int n = 0; n <= max_code; ++n) {
        const int l = len[n];
        if (l) code[n] = (uint16_t)bi_reverse(next[l]++, l);
    }
}

// tr_static_init's static trees
C3B_HD void static_trees(Trees &t) {
    for (int b = 0; b <= MAX_BITS; ++b) t.bl_count[b] = 0;
    for (int n = 0; n < 288; ++n) {
        t.s_llen[n] = (uint8_t)(n < 144 ? 8 : n < 256 ? 9 : n < 280 ? 7 : 8);
        t.bl_count[t.s_llen[n]]++;
    }
    gen_codes(t.s_lcode, t.s_llen, 287, t.bl_count);
    for (int n = 0; n < D_CODES; ++n) {
        t.s_dlen[n] = 5;
        t.s_dcode[n] = (uint16_t)bi_reverse((unsigned)n, 5);
    }
}

// What comes before Deflater::run(len) on a compressor's window, head and prev, which may hold whatever an earlier block left
// there: the payload into window[0 .. len), fill_window's high-water zeroing of the 258 bytes past it (as far as the window
// goes), and head emptied.  prev is zeroed too, though zlib's is not: no entry of prev is read before it is written.  Thread
// tid of nthreads does its share (the kernel's CTA: tid of Z_THREADS, then a barrier; the host build: 0 of 1).  head and prev
// are zeroed a 32-bit word at a time, so both must be 4-byte aligned.
C3B_HD void reset_block(uint8_t *window, uint16_t *head, uint16_t *prev, const uint8_t *src, int len, int tid, int nthreads) {
    for (int i = tid; i < len; i += nthreads) window[i] = src[i];
    const int zend = len + WIN_INIT < WINDOW ? len + WIN_INIT : WINDOW;
    for (int i = len + tid; i < zend; i += nthreads) window[i] = 0;
    uint32_t *h = reinterpret_cast<uint32_t *>(head), *p = reinterpret_cast<uint32_t *>(prev);
    for (int i = tid; i < W_SIZE / 2; i += nthreads) h[i] = 0, p[i] = 0;      // head: 2^15 entries (hash_bits 15), prev: W_SIZE
}

// The compressor of one block.  window: WINDOW bytes, head / prev: 32 Ki entries each, sym: SYM_END bytes; out: cap bytes.
struct Deflater {
    uint8_t *window;
    uint16_t *head, *prev;
    uint8_t *sym;
    Trees *t;
    uint8_t *out;
    int cap, pos;
    uint64_t bb;
    int bv;
    bool overflow;
    unsigned strstart, lookahead, match_start, prev_match, match_length, prev_length, ins_h, sym_next;
    long block_start;
    int match_available;
    unsigned long opt_len, static_len;
    Tree L, D, BL;
    int seen[5];                        // stored, fixed and dynamic blocks, gen_bitlen overflow repairs, window slides

    // ---- the bit buffer: LSB first, as send_bits packs it
    C3B_HD void put_byte(unsigned b) {
        if (pos < cap) out[pos] = (uint8_t)b;
        else overflow = true;
        ++pos;
    }
    C3B_HD void send_bits(unsigned value, int length) {
        bb |= (uint64_t)value << bv;
        bv += length;
        while (bv >= 8) {
            put_byte((unsigned)(bb & 0xff));
            bb >>= 8;
            bv -= 8;
        }
    }
    C3B_HD void bi_windup() {
        if (bv > 0) put_byte((unsigned)(bb & 0xff));
        bb = 0;
        bv = 0;
    }

    // ---- trees.c
    C3B_HD void init_block() {
        for (int n = 0; n < L_CODES; ++n) t->l.freq[n] = 0;
        for (int n = 0; n < D_CODES; ++n) t->d.freq[n] = 0;
        for (int n = 0; n < BL_CODES; ++n) t->bl.freq[n] = 0;
        t->l.freq[END_BLOCK] = 1;
        opt_len = static_len = 0;
        sym_next = 0;
    }
    C3B_HD bool tally(unsigned dist, unsigned lc) {
        sym[sym_next++] = (uint8_t)dist;
        sym[sym_next++] = (uint8_t)(dist >> 8);
        sym[sym_next++] = (uint8_t)lc;
        if (dist == 0) {
            t->l.freq[lc]++;
        } else {
            dist--;
            t->l.freq[length_code(lc) + END_BLOCK + 1]++;
            t->d.freq[dist_code(dist)]++;
        }
        return sym_next == (unsigned)SYM_END;
    }
    C3B_HD int extra_of(const Tree &tr, int n) const {
        const int c = n - tr.extra_base;
        return tr.kind == 0 ? lextra(c) : tr.kind == 1 ? dextra(c) : blextra(c);
    }
    C3B_HD bool smaller(const Tree &tr, int n, int m) const {
        return tr.freq[n] < tr.freq[m] || (tr.freq[n] == tr.freq[m] && t->depth[n] <= t->depth[m]);
    }
    C3B_HD void pqdownheap(const Tree &tr, int k) {
        int16_t *heap = t->heap;
        const int v = heap[k];
        int j = k << 1;
        while (j <= t->heap_len) {
            if (j < t->heap_len && smaller(tr, heap[j + 1], heap[j])) j++;
            if (smaller(tr, v, heap[j])) break;
            heap[k] = heap[j];
            k = j;
            j <<= 1;
        }
        heap[k] = (int16_t)v;
    }
    C3B_HD void gen_bitlen(Tree &tr) {
        int16_t *heap = t->heap;
        uint16_t *bl_count = t->bl_count;
        int overflow_n = 0;
        for (int bits = 0; bits <= MAX_BITS; ++bits) bl_count[bits] = 0;
        tr.len[heap[t->heap_max]] = 0;                                  // the root
        int h;
        for (h = t->heap_max + 1; h < HEAP_SIZE; ++h) {
            const int n = heap[h];
            int bits = tr.len[tr.dad[n]] + 1;
            if (bits > tr.max_length) bits = tr.max_length, overflow_n++;
            tr.len[n] = (uint16_t)bits;
            if (n > tr.max_code) continue;                              // not a leaf
            bl_count[bits]++;
            const int xbits = n >= tr.extra_base ? extra_of(tr, n) : 0;
            const unsigned f = tr.freq[n];
            opt_len += (unsigned long)f * (unsigned)(bits + xbits);
            if (tr.static_len) static_len += (unsigned long)f * (unsigned)(tr.static_len[n] + xbits);
        }
        if (overflow_n == 0) return;
        seen[3]++;
        do {
            int bits = tr.max_length - 1;
            while (bl_count[bits] == 0) bits--;
            bl_count[bits]--;
            bl_count[bits + 1] += 2;
            bl_count[tr.max_length]--;
            overflow_n -= 2;
        } while (overflow_n > 0);
        for (int bits = tr.max_length; bits != 0; bits--) {
            int n = bl_count[bits];
            while (n != 0) {
                const int m = heap[--h];
                if (m > tr.max_code) continue;
                if (tr.len[m] != (unsigned)bits) {
                    opt_len += ((unsigned long)bits - tr.len[m]) * tr.freq[m];
                    tr.len[m] = (uint16_t)bits;
                }
                n--;
            }
        }
    }
    C3B_HD void build_tree(Tree &tr) {
        int16_t *heap = t->heap;
        uint8_t *depth = t->depth;
        int max_code = -1, node;
        t->heap_len = 0;
        t->heap_max = HEAP_SIZE;
        for (int n = 0; n < tr.elems; ++n) {
            if (tr.freq[n] != 0) {
                heap[++t->heap_len] = (int16_t)(max_code = n);
                depth[n] = 0;
            } else {
                tr.len[n] = 0;
            }
        }
        // at least two codes of non-zero frequency
        while (t->heap_len < 2) {
            node = heap[++t->heap_len] = (int16_t)(max_code < 2 ? ++max_code : 0);
            tr.freq[node] = 1;
            depth[node] = 0;
            opt_len--;
            if (tr.static_len) static_len -= tr.static_len[node];
        }
        tr.max_code = max_code;
        for (int n = t->heap_len / 2; n >= 1; n--) pqdownheap(tr, n);
        node = tr.elems;
        do {
            const int n = heap[1];                                      // pqremove
            heap[1] = heap[t->heap_len--];
            pqdownheap(tr, 1);
            const int m = heap[1];
            heap[--t->heap_max] = (int16_t)n;
            heap[--t->heap_max] = (int16_t)m;
            tr.freq[node] = (uint16_t)(tr.freq[n] + tr.freq[m]);
            depth[node] = (uint8_t)((depth[n] >= depth[m] ? depth[n] : depth[m]) + 1);
            tr.dad[n] = tr.dad[m] = (uint16_t)node;
            heap[1] = (int16_t)node++;
            pqdownheap(tr, 1);
        } while (t->heap_len >= 2);
        heap[--t->heap_max] = heap[1];
        gen_bitlen(tr);
        gen_codes(tr.code, tr.len, max_code, t->bl_count);
    }
    C3B_HD void scan_tree(Tree &tr, int max_code) {
        uint16_t *blf = t->bl.freq;
        int prevlen = -1, nextlen = tr.len[0], count = 0, max_count = 7, min_count = 4;
        if (nextlen == 0) max_count = 138, min_count = 3;
        tr.len[max_code + 1] = 0xffff;                                  // guard
        for (int n = 0; n <= max_code; n++) {
            const int curlen = nextlen;
            nextlen = tr.len[n + 1];
            if (++count < max_count && curlen == nextlen) {
                continue;
            } else if (count < min_count) {
                blf[curlen] = (uint16_t)(blf[curlen] + count);
            } else if (curlen != 0) {
                if (curlen != prevlen) blf[curlen]++;
                blf[REP_3_6]++;
            } else if (count <= 10) {
                blf[REPZ_3_10]++;
            } else {
                blf[REPZ_11_138]++;
            }
            count = 0;
            prevlen = curlen;
            if (nextlen == 0) max_count = 138, min_count = 3;
            else if (curlen == nextlen) max_count = 6, min_count = 3;
            else max_count = 7, min_count = 4;
        }
    }
    C3B_HD void send_code(int c, const Tree &tr) { send_bits(tr.code[c], tr.len[c]); }
    C3B_HD void send_tree(const Tree &tr, int max_code) {
        int prevlen = -1, nextlen = tr.len[0], count = 0, max_count = 7, min_count = 4;
        if (nextlen == 0) max_count = 138, min_count = 3;
        for (int n = 0; n <= max_code; n++) {
            const int curlen = nextlen;
            nextlen = tr.len[n + 1];
            if (++count < max_count && curlen == nextlen) {
                continue;
            } else if (count < min_count) {
                do { send_code(curlen, BL); } while (--count != 0);
            } else if (curlen != 0) {
                if (curlen != prevlen) {
                    send_code(curlen, BL);
                    count--;
                }
                send_code(REP_3_6, BL);
                send_bits((unsigned)(count - 3), 2);
            } else if (count <= 10) {
                send_code(REPZ_3_10, BL);
                send_bits((unsigned)(count - 3), 3);
            } else {
                send_code(REPZ_11_138, BL);
                send_bits((unsigned)(count - 11), 7);
            }
            count = 0;
            prevlen = curlen;
            if (nextlen == 0) max_count = 138, min_count = 3;
            else if (curlen == nextlen) max_count = 6, min_count = 3;
            else max_count = 7, min_count = 4;
        }
    }
    // bl_order: the order RFC 1951 sends the bit-length code lengths in
    C3B_HD static int bl_order(int r) { return "\x10\x11\x12\x00\x08\x07\x09\x06\x0a\x05\x0b\x04\x0c\x03\x0d\x02\x0e\x01\x0f"[r]; }
    C3B_HD int build_bl_tree() {
        scan_tree(L, L.max_code);
        scan_tree(D, D.max_code);
        build_tree(BL);
        int max_blindex;
        for (max_blindex = BL_CODES - 1; max_blindex >= 3; max_blindex--)
            if (BL.len[bl_order(max_blindex)] != 0) break;
        opt_len += 3 * ((unsigned long)max_blindex + 1) + 5 + 5 + 4;
        return max_blindex;
    }
    // compress_block with the dynamic trees (stat = false) or the static ones
    C3B_HD void compress_block(bool stat) {
        for (unsigned sx = 0; sx < sym_next; sx += 3) {
            unsigned dist = sym[sx] | (unsigned)sym[sx + 1] << 8;
            unsigned lc = sym[sx + 2];
            if (dist == 0) {
                if (stat) send_bits(t->s_lcode[lc], t->s_llen[lc]);
                else send_code((int)lc, L);
                continue;
            }
            int code = length_code(lc);
            const int sc = code + END_BLOCK + 1;
            if (stat) send_bits(t->s_lcode[sc], t->s_llen[sc]);
            else send_code(sc, L);
            int extra = lextra(code);
            if (extra) send_bits(lc - base_length(code), extra);
            dist--;
            code = dist_code(dist);
            if (stat) send_bits(t->s_dcode[code], t->s_dlen[code]);
            else send_code(code, D);
            extra = dextra(code);
            if (extra) send_bits(dist - base_dist(code), extra);
        }
        if (stat) send_bits(t->s_lcode[END_BLOCK], t->s_llen[END_BLOCK]);
        else send_code(END_BLOCK, L);
    }
    C3B_HD void flush_block(bool last) {
        const uint8_t *buf = block_start >= 0 ? window + block_start : nullptr;
        const unsigned long stored_len = (unsigned long)((long)strstart - block_start);
        build_tree(L);
        build_tree(D);
        const int max_blindex = build_bl_tree();
        unsigned long opt_lenb = (opt_len + 3 + 7) >> 3;
        const unsigned long static_lenb = (static_len + 3 + 7) >> 3;
        if (static_lenb <= opt_lenb) opt_lenb = static_lenb;
        if (stored_len + 4 <= opt_lenb && buf) {
            seen[0]++;
            send_bits(last ? 1u : 0u, 3);                               // STORED_BLOCK << 1 | last
            bi_windup();
            put_byte(stored_len & 0xff);
            put_byte((stored_len >> 8) & 0xff);
            put_byte(~stored_len & 0xff);
            put_byte((~stored_len >> 8) & 0xff);
            for (unsigned long i = 0; i < stored_len; ++i) put_byte(buf[i]);
        } else if (static_lenb == opt_lenb) {
            seen[1]++;
            send_bits(2u + (last ? 1u : 0u), 3);                        // STATIC_TREES << 1 | last
            compress_block(true);
        } else {
            seen[2]++;
            send_bits(4u + (last ? 1u : 0u), 3);                        // DYN_TREES << 1 | last
            const int lcodes = L.max_code + 1, dcodes = D.max_code + 1, blcodes = max_blindex + 1;
            send_bits((unsigned)(lcodes - 257), 5);
            send_bits((unsigned)(dcodes - 1), 5);
            send_bits((unsigned)(blcodes - 4), 4);
            for (int r = 0; r < blcodes; ++r) send_bits(BL.len[bl_order(r)], 3);
            send_tree(L, lcodes - 1);
            send_tree(D, dcodes - 1);
            compress_block(false);
        }
        init_block();
        if (last) bi_windup();
        block_start = (long)strstart;                                   // FLUSH_BLOCK_ONLY
    }

    // ---- deflate.c
    C3B_HD void update_hash(unsigned c) { ins_h = ((ins_h << HASH_SHIFT) ^ c) & HASH_MASK; }
    C3B_HD unsigned insert_string(unsigned str) {
        update_hash(window[str + (MIN_MATCH - 1)]);
        const unsigned h = head[ins_h];
        prev[str & W_MASK] = (uint16_t)h;
        head[ins_h] = (uint16_t)str;
        return h;
    }
    // fill_window once all input is in the window: only the slide can happen
    C3B_HD void fill_window() {
        const unsigned more = (unsigned)(WINDOW - lookahead - strstart);
        if (strstart >= (unsigned)(W_SIZE + MAX_DIST)) {
            seen[4]++;
            for (unsigned i = 0; i < (unsigned)W_SIZE - more; ++i) window[i] = window[i + W_SIZE];
            match_start -= W_SIZE;
            strstart -= W_SIZE;
            block_start -= W_SIZE;
            for (int n = 0; n < 32768; ++n) head[n] = (uint16_t)(head[n] >= W_SIZE ? head[n] - W_SIZE : 0);
            for (int n = 0; n < W_SIZE; ++n) prev[n] = (uint16_t)(prev[n] >= W_SIZE ? prev[n] - W_SIZE : 0);
        }
    }
    C3B_HD unsigned longest_match(unsigned cur_match) {
        unsigned chain_length = CHAIN;
        const uint8_t *scan = window + strstart;
        int best_len = (int)prev_length;
        int nice_match = (int)NICE;
        const unsigned limit = strstart > (unsigned)MAX_DIST ? strstart - MAX_DIST : 0;
        const uint8_t *strend = window + strstart + MAX_MATCH;
        uint8_t scan_end1 = scan[best_len - 1], scan_end = scan[best_len];
        if (prev_length >= GOOD) chain_length >>= 2;
        if ((unsigned)nice_match > lookahead) nice_match = (int)lookahead;
        do {
            const uint8_t *match = window + cur_match;
            if (match[best_len] != scan_end || match[best_len - 1] != scan_end1 || match[0] != scan[0] || match[1] != scan[1])
                continue;
            // scan[2] and match[2] are equal when the rest match: the hash keys are equal and hash_bits >= 8
            const uint8_t *s = scan + 2, *m = match + 2;
            while (*++s == *++m && s < strend) {}
            const int len = MAX_MATCH - (int)(strend - s);
            if (len > best_len) {
                match_start = cur_match;
                best_len = len;
                if (len >= nice_match) break;
                scan_end1 = scan[best_len - 1];
                scan_end = scan[best_len];
            }
        } while ((cur_match = prev[cur_match & W_MASK]) > limit && --chain_length != 0);
        return (unsigned)best_len <= lookahead ? (unsigned)best_len : lookahead;
    }

    // The stream of window[0 .. n), after reset_block.  Returns the bytes written to out, or -1 past cap.
    C3B_HD int run(int n) {
        L = Tree{t->l.freq, t->l.dad, t->l.len, t->l.code, L_CODES, END_BLOCK + 1, MAX_BITS, 0, 0, t->s_llen};
        D = Tree{t->d.freq, t->d.dad, t->d.len, t->d.code, D_CODES, 0, MAX_BITS, 0, 1, t->s_dlen};
        BL = Tree{t->bl.freq, t->bl.dad, t->bl.len, t->bl.code, BL_CODES, 0, MAX_BL_BITS, 0, 2, nullptr};
        static_trees(*t);
        pos = 0, bb = 0, bv = 0, overflow = false;
        for (int i = 0; i < 5; ++i) seen[i] = 0;
        strstart = 0, block_start = 0, match_start = prev_match = 0, ins_h = 0;
        match_length = prev_length = MIN_MATCH - 1;
        match_available = 0;
        init_block();
        // the first fill_window reads the whole payload
        lookahead = (unsigned)n;
        if (lookahead >= (unsigned)MIN_MATCH) {
            ins_h = window[0];
            update_hash(window[1]);
        }
        for (;;) {
            if (lookahead < (unsigned)MIN_LOOKAHEAD) {
                fill_window();
                if (lookahead == 0) break;
            }
            unsigned hash_head = 0;
            if (lookahead >= (unsigned)MIN_MATCH) hash_head = insert_string(strstart);
            prev_length = match_length, prev_match = match_start;
            match_length = MIN_MATCH - 1;
            if (hash_head != 0 && prev_length < LAZY && strstart - hash_head <= (unsigned)MAX_DIST) {
                match_length = longest_match(hash_head);
                if (match_length == (unsigned)MIN_MATCH && strstart - match_start > (unsigned)TOO_FAR) match_length = MIN_MATCH - 1;
            }
            if (prev_length >= (unsigned)MIN_MATCH && match_length <= prev_length) {
                const unsigned max_insert = strstart + lookahead - MIN_MATCH;
                const bool bflush = tally(strstart - 1 - prev_match, prev_length - MIN_MATCH);
                lookahead -= prev_length - 1;
                prev_length -= 2;
                do {
                    if (++strstart <= max_insert) insert_string(strstart);
                } while (--prev_length != 0);
                match_available = 0;
                match_length = MIN_MATCH - 1;
                strstart++;
                if (bflush) flush_block(false);
            } else if (match_available) {
                if (tally(0, window[strstart - 1])) flush_block(false);
                strstart++;
                lookahead--;
            } else {
                match_available = 1;
                strstart++;
                lookahead--;
            }
        }
        if (match_available) {
            tally(0, window[strstart - 1]);
            match_available = 0;
        }
        flush_block(true);
        return overflow ? -1 : pos;
    }
};

// The 18 header bytes of a BGZF block whose DEFLATE stream is clen bytes (bam_io._bgzf_block: gzip with FEXTRA, MTIME 0, XFL 0,
// OS 255, and the BC subfield holding the block's total size - 1).
C3B_HD void bgzf_header(uint8_t *h, int clen) {
    const int bsize = clen + HEADER + FOOTER - 1;
    const uint8_t fixed[16] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 0x42, 0x43, 2, 0};
    for (int i = 0; i < 16; ++i) h[i] = fixed[i];
    h[16] = (uint8_t)(bsize & 0xff);
    h[17] = (uint8_t)(bsize >> 8);
}
C3B_HD void put32(uint8_t *p, uint32_t v) {
    p[0] = (uint8_t)v, p[1] = (uint8_t)(v >> 8), p[2] = (uint8_t)(v >> 16), p[3] = (uint8_t)(v >> 24);
}

}  // namespace c3b_deflate
