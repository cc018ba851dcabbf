// deflate_host.cpp - a host build of clair3_b200/csrc/deflate.cuh for tests/test_deflate_host_cpu.py, compiled there with
// AddressSanitizer and UBSan.  The window, head, prev and symbol buffer are exact-size heap allocations of the sizes the GPU
// kernel gives them, and the output buffer is exactly the BGZF block bound, so a read or write past any of them is a sanitizer
// report.
//
//   deflate_host bgzf < cases > blocks     cases: {u32 n, n bytes}...; blocks: {i32 size, size bytes}... - each payload as one
//                                          whole BGZF block (bgzf_deflate_kernel's bytes), its CRC-32 from the 32-lane split;
//                                          size -1: the stream did not fit the block
//   deflate_host seen < cases > counts     cases as above; per case five i32: the stored, fixed and dynamic blocks of its stream,
//                                          gen_bitlen's overflow repairs and fill_window's slides
//   deflate_host cta K < cases > blocks    as bgzf, but as K CTAs of bgzf_deflate_kernel run them: K compressor states allocated
//                                          once and every byte of them filled with a seeded non-zero pattern, payload i on state
//                                          i % K after what payload i - K left there, with the kernel's reset_block between
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "deflate.cuh"

using namespace c3b_deflate;

static bool get32(uint32_t *v) { return fread(v, 4, 1, stdin) == 1; }

// One CTA's compressor state: what the kernel keeps in shared memory and its global symbol-buffer slot, and its output slot.
struct State {
    uint8_t *window = new uint8_t[WINDOW];
    uint16_t *head = new uint16_t[32768], *prev = new uint16_t[W_SIZE];
    uint8_t *sym = new uint8_t[SYM_END];
    Trees *t = new Trees;
    uint8_t *block = new uint8_t[BLOCK_MAX];
    ~State() {
        delete[] block;
        delete t;
        delete[] sym;
        delete[] prev;
        delete[] head;
        delete[] window;
    }
    void poison(uint32_t &x) {
        auto fill = [&x](void *p, size_t n) {
            uint8_t *b = static_cast<uint8_t *>(p);
            for (size_t i = 0; i < n; ++i) {
                x ^= x << 13, x ^= x >> 17, x ^= x << 5;             // xorshift32
                b[i] = (uint8_t)(x >> 24) ? (uint8_t)(x >> 24) : 0xA5;
            }
        };
        fill(window, WINDOW), fill(head, 32768 * 2), fill(prev, W_SIZE * 2), fill(sym, SYM_END), fill(t, sizeof(Trees));
        fill(block, BLOCK_MAX);
    }
};

// src as one BGZF block in s.block, as bgzf_deflate_kernel frames it: its size, or -1 when the stream does not fit the block.
static int32_t compress(State &s, const uint32_t *tab, const uint8_t *src, uint32_t n, int *seen) {
    reset_block(s.window, s.head, s.prev, src, (int)n, 0, 1);
    Deflater z;
    z.window = s.window;
    z.head = s.head;
    z.prev = s.prev;
    z.sym = s.sym;
    z.t = s.t;
    z.out = s.block + HEADER;
    z.cap = BLOCK_MAX - HEADER - FOOTER;
    const int clen = z.run((int)n);
    memcpy(seen, z.seen, sizeof z.seen);
    if (clen < 0) return -1;
    uint32_t x = 0;
    for (int l = 0; l < 32; ++l) x ^= c3b_inflate::crc_lane_term(tab, src, (int)n, l);
    bgzf_header(s.block, clen);
    put32(s.block + HEADER + clen, c3b_inflate::crc_lanes_done(x, (int)n));
    put32(s.block + HEADER + clen + 4, n);
    return HEADER + clen + FOOTER;
}

int main(int argc, char **argv) {
    const bool cta = argc == 3 && !strcmp(argv[1], "cta");
    if (!cta && (argc != 2 || (strcmp(argv[1], "bgzf") && strcmp(argv[1], "seen")))) return 2;
    const bool seen = !strcmp(argv[1], "seen");
    const int k = cta ? atoi(argv[2]) : 0;
    if (cta && k < 1) return 2;
    uint32_t tab[256];
    for (uint32_t i = 0; i < 256; ++i) tab[i] = c3b_inflate::crc_table_entry(i);
    std::vector<State *> states;
    uint32_t x = 0x9E3779B9u;
    for (int c = 0; c < k; ++c) {
        states.push_back(new State);
        states.back()->poison(x);
    }
    uint32_t n;
    for (uint64_t i = 0; get32(&n); ++i) {
        if (n > (uint32_t)PAYLOAD) {
            fprintf(stderr, "payload of %u bytes exceeds a BGZF block's %d\n", n, PAYLOAD);
            return 2;
        }
        uint8_t *src = new uint8_t[n ? n : 1];
        if (n && fread(src, 1, n, stdin) != n) {
            fprintf(stderr, "short input\n");
            return 2;
        }
        State *fresh = cta ? nullptr : new State;     // bgzf / seen: new buffers for every payload
        State &s = cta ? *states[i % k] : *fresh;
        int counts[5];
        const int32_t size = compress(s, tab, src, n, counts);
        if (seen) {
            fwrite(counts, 4, 5, stdout);
        } else {
            fwrite(&size, 4, 1, stdout);
            if (size > 0) fwrite(s.block, 1, (size_t)size, stdout);
        }
        delete fresh;
        delete[] src;
    }
    for (State *s : states) delete s;
    return 0;
}
