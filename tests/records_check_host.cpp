// records_check_host.cpp - a host build of clair3_b200/csrc/records_check.cuh for tests/test_records_check_cpu.py, compiled there
// with AddressSanitizer and UBSan.  Every array is its own exact-size heap allocation, so a read past the n_reads per-read
// entries, the n_reads + 1 offsets or a value array is a sanitizer report.
//
//   records_check_host < cases > verdicts
//   case:    i64 n_reads, u32 present, u32 0, i64 len[5], i64 pos[n], i32 l_qseq[n], then i64 off[n + 1] for each offset array
//            present, in the order cigar, seq, qual, qname, mv.  present: bit f = offset array f, bit 8 + f = its values.
//   verdict: one line per case, "<reason> <read>": 0 0 for records the check passes.
#include <cstdio>
#include <cstdlib>

#include "records_check.cuh"

template <class T> static T *read_array(int64_t n) {
    T *p = new T[n > 0 ? n : 1];
    if (n > 0 && fread(p, sizeof(T), (size_t)n, stdin) != (size_t)n) {
        fprintf(stderr, "short input\n");
        exit(2);
    }
    return p;
}

template <class T> static const T *values(uint32_t present, int f, int64_t len) {
    return present >> (8 + f) & 1 ? new T[len > 0 ? len : 1]() : nullptr;
}

int main() {
    int64_t n;
    while (fread(&n, 8, 1, stdin) == 1) {
        uint32_t hdr[2];
        int64_t len[5];
        if (fread(hdr, 4, 2, stdin) != 2 || fread(len, 8, 5, stdin) != 5) return 2;
        const uint32_t present = hdr[0];
        int64_t *pos = read_array<int64_t>(n);
        int32_t *l_qseq = read_array<int32_t>(n);
        int64_t *off[5] = {};
        for (int f = 0; f < 5; ++f)
            if (present >> f & 1) off[f] = read_array<int64_t>(n + 1);
        uint16_t *flag = new uint16_t[n > 0 ? n : 1]();
        uint8_t *mapq = new uint8_t[n > 0 ? n : 1]();
        c3b_fa_records r = {};
        c3b_bam_records &c = r.core;
        c.n_reads = n;
        c.pos = pos; c.flag = flag; c.mapq = mapq; c.l_qseq = l_qseq;
        c.cigar_off = off[0]; c.cigar = values<uint32_t>(present, 0, len[0]); c.n_cigar = len[0];
        c.seq_off = off[1]; c.seq = values<uint8_t>(present, 1, len[1]); c.n_seq = len[1];
        r.qual_off = off[2]; r.qual = values<uint8_t>(present, 2, len[2]); r.n_qual = len[2];
        r.qname_off = off[3]; r.qname = values<uint8_t>(present, 3, len[3]); r.n_qname = len[3];
        r.mv_off = off[4]; r.mv = values<int32_t>(present, 4, len[4]); r.n_mv = len[4];
        const bool opt = (present & 0x1c1c) != 0;
        const uint64_t key = c3b_records_check(&c, opt ? &r : nullptr);
        if (key == C3B_REC_OK) printf("0 0\n");
        else printf("%llu %lld\n", (unsigned long long)(key >> 40), (long long)c3b_records_fault_read(key));
        delete[] c.cigar;
        delete[] c.seq;
        delete[] r.qual;
        delete[] r.qname;
        delete[] r.mv;
        for (int f = 0; f < 5; ++f) delete[] off[f];
        delete[] flag;
        delete[] mapq;
        delete[] l_qseq;
        delete[] pos;
    }
    return 0;
}
