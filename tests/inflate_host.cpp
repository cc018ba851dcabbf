// inflate_host.cpp - a host build of clair3_b200/csrc/inflate.cuh for tests/test_inflate_host_cpu.py, compiled there with
// AddressSanitizer and UBSan.  Every buffer is its own exact-size heap allocation, so a read or write past a stream, an output
// capacity or a table is a sanitizer report.
//
//   inflate_host inflate < cases > results    cases: {u32 n_in, u32 cap, n_in bytes}...; results: {i32 status, i32 n_out, bytes}...
//   inflate_host crc < cases                  cases: {u32 n, u32 k, n bytes}...; one line per case, in hex:
//                                             the CRC-32 from crc_shift(~0, n) and R(0, data); from R(~0, data[:k]) shifted past
//                                             data[k:]; and from the 32-lane split of bam_decode.cu's bam_inflate_kernel
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "inflate.cuh"

using namespace c3b_inflate;

static bool get32(uint32_t *v) { return fread(v, 4, 1, stdin) == 1; }

static uint8_t *read_exact(uint32_t n) {
    uint8_t *p = new uint8_t[n ? n : 1];
    if (n && fread(p, 1, n, stdin) != n) {
        fprintf(stderr, "short input\n");
        exit(2);
    }
    return p;
}

int main(int argc, char **argv) {
    if (argc != 2) return 2;
    if (!strcmp(argv[1], "inflate")) {
        uint32_t n_in, cap;
        while (get32(&n_in) && get32(&cap)) {
            uint8_t *in = read_exact(n_in);
            uint8_t *out = new uint8_t[cap ? cap : 1];
            Tables *t = new Tables;
            int n_out = -1;
            const int32_t st = inflate(in, (int)n_in, out, (int)cap, &n_out, *t);
            fwrite(&st, 4, 1, stdout);
            fwrite(&n_out, 4, 1, stdout);
            fwrite(out, 1, n_out > 0 ? n_out : 0, stdout);
            delete t;
            delete[] out;
            delete[] in;
        }
        return 0;
    }
    if (!strcmp(argv[1], "crc")) {
        uint32_t tab[256];
        for (uint32_t i = 0; i < 256; ++i) tab[i] = crc_table_entry(i);
        uint32_t n, k;
        while (get32(&n) && get32(&k)) {
            uint8_t *p = read_exact(n);
            const uint32_t whole = ~(crc_shift(0xffffffffu, n) ^ crc_update(tab, 0, p, (int)n));
            const uint32_t split = ~(crc_shift(crc_update(tab, 0xffffffffu, p, (int)k), n - k) ^ crc_update(tab, 0, p + k, (int)(n - k)));
            // the lanes of bam_inflate_kernel: lane l takes [l * chunk, min((l + 1) * chunk, n)) and shifts it past the rest
            const int chunk = ((int)n + 31) / 32;
            uint32_t lanes = 0;
            for (int l = 0; l < 32; ++l) {
                const int a = l * chunk, e = a + chunk < (int)n ? a + chunk : (int)n;
                if (a < e) lanes ^= crc_shift(crc_update(tab, 0, p + a, e - a), (uint32_t)((int)n - e));
            }
            lanes = ~(lanes ^ crc_shift(0xffffffffu, n));
            printf("%08x %08x %08x\n", whole, split, lanes);
            delete[] p;
        }
        return 0;
    }
    return 2;
}
