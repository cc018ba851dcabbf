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
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "deflate.cuh"

using namespace c3b_deflate;

static bool get32(uint32_t *v) { return fread(v, 4, 1, stdin) == 1; }

int main(int argc, char **argv) {
    if (argc != 2 || (strcmp(argv[1], "bgzf") && strcmp(argv[1], "seen"))) return 2;
    const bool seen = !strcmp(argv[1], "seen");
    uint32_t tab[256];
    for (uint32_t i = 0; i < 256; ++i) tab[i] = c3b_inflate::crc_table_entry(i);
    uint32_t n;
    while (get32(&n)) {
        if (n > (uint32_t)PAYLOAD) {
            fprintf(stderr, "payload of %u bytes exceeds a BGZF block's %d\n", n, PAYLOAD);
            return 2;
        }
        uint8_t *src = new uint8_t[n ? n : 1];
        if (n && fread(src, 1, n, stdin) != n) {
            fprintf(stderr, "short input\n");
            return 2;
        }
        Deflater z;
        z.window = new uint8_t[WINDOW];
        z.head = new uint16_t[32768];
        z.prev = new uint16_t[W_SIZE];
        z.sym = new uint8_t[SYM_END];
        z.t = new Trees;
        uint8_t *block = new uint8_t[BLOCK_MAX];
        // what the kernel's threads do before the compressor starts
        memcpy(z.window, src, n);
        memset(z.window + n, 0, (size_t)(n + WIN_INIT < (uint32_t)WINDOW ? WIN_INIT : WINDOW - n));
        memset(z.head, 0, 32768 * sizeof(uint16_t));
        memset(z.prev, 0, W_SIZE * sizeof(uint16_t));
        z.out = block + HEADER;
        z.cap = BLOCK_MAX - HEADER - FOOTER;
        const int clen = z.run((int)n);
        int32_t size = -1;
        if (clen >= 0) {
            uint32_t x = 0;
            for (int l = 0; l < 32; ++l) x ^= c3b_inflate::crc_lane_term(tab, src, (int)n, l);
            bgzf_header(block, clen);
            put32(block + HEADER + clen, c3b_inflate::crc_lanes_done(x, (int)n));
            put32(block + HEADER + clen + 4, n);
            size = HEADER + clen + FOOTER;
        }
        if (seen) {
            fwrite(z.seen, 4, 5, stdout);
        } else {
            fwrite(&size, 4, 1, stdout);
            if (size > 0) fwrite(block, 1, (size_t)size, stdout);
        }
        delete[] block;
        delete z.t;
        delete[] z.sym;
        delete[] z.prev;
        delete[] z.head;
        delete[] z.window;
        delete[] src;
    }
    return 0;
}
