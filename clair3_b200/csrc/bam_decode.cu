// bam_decode.cu - the BAM reader on the GPU (include/clair3_b200_bam.h): whole BGZF blocks in, one region's alignment records
// out, in the c3b_fa_records layout the pileup counter and the full-alignment builder read.
//
// The SAM/BAM specification (section 4) fixes the format: a BAM file is a series of BGZF blocks, each a gzip member of at most
// 64 KiB whose extra field's BC subfield gives its compressed size and whose footer gives the CRC-32 and size of its payload; the
// uncompressed stream is the header and then the records, each an int32 block_size and that many bytes.  The host checks the
// block headers, computes every block's output offset from the ISIZE footers and uploads the bytes; then, on one stream:
//
//   B1 bam_inflate      one WARP per BGZF block: lane 0 inflates the block (inflate.cuh) into shared memory, the warp copies it
//                       to its offset in the uncompressed buffer and checks its CRC-32 and size.  A bad block sets its status.
//   B2 bam_speculate    one warp per block: the first offset of the block that passes the necessary conditions of a record header
//                       (block_size holds the fields the header declares, a printable name ending in NUL, ...); lane 0 chases
//                       block_size from there to the end of the block, marking every offset it visits.
//   B3 bam_fixup        one thread: walks the blocks in order carrying the true chain from first_uoff.  Where the true entry
//                       into a block is marked, the two chains coincide from there on (a chain is determined by its offset), so
//                       it jumps to the speculative chain's exit; otherwise it chases until it meets a marked offset or leaves the
//                       block.  Checks that the chain ends exactly at end_uoff.
//   B4 bam_starts       one warp per block: clears the marks before the point where the true chain met the speculative one,
//                       re-marks the true chain there, and counts the block's record starts.  The marks are then exactly the
//                       true chain: the speculation decides where work starts, never the result.
//   B5 block scan       record index of each block's first record; the total is the number of records.
//   B6 bam_offsets      one warp per block: the offset of every record, in file order, and the first record that ends the run
//                       (a later contig, or pos >= end: read_bam's "stop" conditions), min-reduced.
//   B7 bam_parse        one thread per record: checks block_size against the fields, applies the filter below the first stop,
//                       walks the aux fields for mv (with fa_fields) and for the CG tag of a placeholder CIGAR (read_bam's
//                       _cg_cigar), sums the reference span of the real CIGAR and writes the kept record's counts.
//   B8 block scans      record index, CIGAR words, sequence bytes (and qualities, names, mv values) of each kept record.
//   B9 bam_scatter      one warp per kept record: every array into the packed outputs.
//
// c3b_fasta_fetch reuses the upload and B1 for the blocks of a bgzip-compressed FASTA window, then gathers the window's bases
// with one thread each, skipping the line ends by arithmetic; c3b_fasta_status reads its bad-block word.
//
// The BGZF writer runs the other direction on the same workspace and upload (c3b_bgzf_compress):
//   Z1 bgzf_deflate     one CTA per SM, striding over the 0xFF00-byte payloads: the CTA loads a payload into its shared
//                       window, thread 0 compresses it exactly as zlib level 6 does (deflate.cuh) into the block's
//                       64 KiB slot, warp 1 computes its CRC-32 with bam_inflate's lane split, and thread 0 frames the block.
//   Z2 block scan       each block's offset in the file from the compressed sizes, and the file size.
//   Z3 bgzf_pack        one CTA per block: the slots into one contiguous file image.
//
// The only host wait is c3b_bam_sizes, after the totals.  Every buffer is sized from what the host knows before the decode: the
// compressed bytes and the sum of ISIZE (U): a record takes at least 36 bytes of U, so there are at most U / 36 + 1 records, and
// every value array holds at most U entries.  Valid input never reaches a capacity; malformed input is bounds-checked at every
// read of U and every write.
#include <limits.h>
#include <string.h>

#include <vector>

#include "block_scan.cuh"
#include "c3b_internal.h"
#include "deflate.cuh"
#include "inflate.cuh"
#include "../../include/clair3_b200_bam.h"

namespace {

using namespace c3b_inflate;

// One BGZF block as the host found it in the uploaded bytes.
struct Block {
    int64_t coff;       // first byte of the DEFLATE payload in the uploaded bytes
    int64_t uoff;       // first byte of the block's output in the uncompressed buffer
    int32_t clen;       // payload bytes
    int32_t isize;      // ISIZE
    uint32_t crc;       // CRC32
    int32_t pad;
};

constexpr int REC_MIN = 36;                 // block_size field + the 32-byte core
constexpr int WARPS = 8;                    // warps per CTA of the per-record warp kernels

// counter words: 0 (block << 4 | status) of the first bad block, 1 the first record that ends the run, 2 (record << 4 | error)
// of the first malformed record (these three start at all ones: min-reduced), 3 the chain's error, 4 its offset, 5 records,
// 6 kept records, 7..11 CIGAR words, sequence bytes, qualities, name bytes and mv values of the kept records.
constexpr int N_COUNTERS = 12;
enum ChainError : int { CHAIN_OK = 0, CHAIN_TRUNCATED = 1, CHAIN_SHORT_BLOCK_SIZE = 2 };
enum RecordError : int { REC_FIELDS = 1, REC_AUX = 2 };
constexpr uint32_t CG_MAX = 1u << 29;       // htslib's bam_tag2cigar moves a CG tag of fewer words than this

__device__ __forceinline__ uint32_t rd32(const uint8_t *u, int64_t o) {
    return (uint32_t)u[o] | (uint32_t)u[o + 1] << 8 | (uint32_t)u[o + 2] << 16 | (uint32_t)u[o + 3] << 24;
}
__device__ __forceinline__ uint32_t rd16(const uint8_t *u, int64_t o) { return (uint32_t)u[o] | (uint32_t)u[o + 1] << 8; }

// The uncompressed range [lo, hi) of block b that can hold record starts.
__device__ __forceinline__ void block_range(const Block &B, int64_t first, int64_t end_u, int64_t &lo, int64_t &hi) {
    lo = B.uoff > first ? B.uoff : first;
    hi = B.uoff + B.isize < end_u ? B.uoff + B.isize : end_u;
}

// The bytes a record's header says its fields take, after block_size; -1 for a header that cannot be a record's.
__device__ __forceinline__ int64_t fields_bytes(const uint8_t *U, int64_t o) {
    const int l_name = U[o + 12], n_cig = (int)rd16(U, o + 16);
    const int32_t l_seq = (int32_t)rd32(U, o + 20);
    if (l_name < 1 || l_seq < 0) return -1;
    return 32 + (int64_t)l_name + 4ll * n_cig + ((int64_t)l_seq + 1) / 2 + l_seq;
}

// Necessary conditions of a record header at o: they only choose where speculation starts.
__device__ bool looks_like_record(const uint8_t *U, int64_t o, int64_t end_u) {
    if (o + REC_MIN > end_u) return false;
    const int32_t bs = (int32_t)rd32(U, o);
    const int64_t need = fields_bytes(U, o);
    if (need < 0 || bs < need || o + 4 + (int64_t)bs > end_u) return false;
    if ((int32_t)rd32(U, o + 4) < -1 || (int32_t)rd32(U, o + 8) < -1 || (int32_t)rd32(U, o + 24) < -1 || (int32_t)rd32(U, o + 28) < -1)
        return false;
    const int l_name = U[o + 12];
    if (U[o + 36 + l_name - 1] != 0) return false;
    for (int i = 0; i < l_name - 1; ++i) {
        const uint8_t c = U[o + 36 + i];
        if (c < 0x21 || c > 0x7e || c == '@') return false;
    }
    return true;
}

// B1
__global__ void __launch_bounds__(32) bam_inflate_kernel(const uint8_t *__restrict__ bytes, const Block *__restrict__ blocks,
                                                         uint8_t *__restrict__ U, unsigned long long *bad) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint8_t *out = smem;                                                   // 64 KiB
    Tables &t = *reinterpret_cast<Tables *>(smem + 65536);
    uint32_t *crc_tab = reinterpret_cast<uint32_t *>(smem + 65536 + (sizeof(Tables) + 15) / 16 * 16);
    const int lane = threadIdx.x, b = blockIdx.x;
    const Block B = blocks[b];
    for (int i = lane; i < 256; i += 32) crc_tab[i] = crc_table_entry(i);
    int st = OK;
    if (lane == 0) {
        int n_out = 0;
        st = inflate(bytes + B.coff, B.clen, out, B.isize, &n_out, t);
        if (st == OK && n_out != B.isize) st = SIZE_MISMATCH;
    }
    st = __shfl_sync(0xffffffffu, st, 0);
    __syncwarp();
    if (st == OK) {
        const int n = B.isize;
        uint8_t *dst = U + B.uoff;
        for (int i = lane; i < n; i += 32) dst[i] = out[i];
        uint32_t term = crc_lane_term(crc_tab, out, n, lane);
        for (int d = 16; d; d >>= 1) term ^= __shfl_xor_sync(0xffffffffu, term, d);
        if (crc_lanes_done(term, n) != B.crc) st = CRC_MISMATCH;
    }
    if (lane == 0 && st != OK) atomicMin(bad, (unsigned long long)b << 4 | (unsigned)st);
}

// B2
__global__ void __launch_bounds__(32) bam_speculate_kernel(const Block *__restrict__ blocks, const uint8_t *__restrict__ U,
                                                           int64_t first, int64_t end_u, uint8_t *__restrict__ mark,
                                                           int64_t *__restrict__ spec_exit) {
    const int lane = threadIdx.x, b = blockIdx.x;
    int64_t lo, hi;
    block_range(blocks[b], first, end_u, lo, hi);
    int64_t s = -1;
    for (int64_t base = lo; base < hi && s < 0; base += 32) {
        const int64_t o = base + lane;
        const unsigned m = __ballot_sync(0xffffffffu, o < hi && looks_like_record(U, o, end_u));
        if (m) s = base + __ffs(m) - 1;
    }
    if (lane != 0) return;
    int64_t o = s;
    if (s >= 0) {
        while (o < hi) {
            if (o + 4 > end_u) { o = -1; break; }
            const int32_t bs = (int32_t)rd32(U, o);
            if (bs < 32) { o = -1; break; }
            mark[o] = 1;
            o += 4 + (int64_t)bs;
        }
    }
    spec_exit[b] = o;                       // the speculative chain's first offset past the block; -1: none, or it broke
}

// B3
__global__ void bam_fixup_kernel(const Block *__restrict__ blocks, int nb, const uint8_t *__restrict__ U, int64_t first,
                                 int64_t end_u, const uint8_t *__restrict__ mark, const int64_t *__restrict__ spec_exit,
                                 int64_t *__restrict__ entry, int64_t *__restrict__ merge, int64_t *counters) {
    int64_t cur = first;
    int err = CHAIN_OK;
    for (int b = 0; b < nb; ++b) {
        int64_t lo, hi;
        block_range(blocks[b], first, end_u, lo, hi);
        entry[b] = merge[b] = -1;
        if (err || cur >= hi) continue;
        entry[b] = cur;
        const int64_t ex = spec_exit[b];
        while (cur < hi && !(mark[cur] && ex >= 0)) {
            if (cur + 4 > end_u) { err = CHAIN_TRUNCATED; break; }
            const int32_t bs = (int32_t)rd32(U, cur);
            if (bs < 32) { err = CHAIN_SHORT_BLOCK_SIZE; break; }
            cur += 4 + (int64_t)bs;
        }
        merge[b] = cur < hi ? cur : hi;
        if (!err && cur < hi) cur = ex;
    }
    if (!err && cur != end_u) err = CHAIN_TRUNCATED;
    counters[3] = err;
    counters[4] = cur;
}

// B4
__global__ void __launch_bounds__(32) bam_starts_kernel(const Block *__restrict__ blocks, const uint8_t *__restrict__ U,
                                                        int64_t first, int64_t end_u, uint8_t *__restrict__ mark,
                                                        const int64_t *__restrict__ entry, const int64_t *__restrict__ merge,
                                                        int32_t *__restrict__ count) {
    const int lane = threadIdx.x, b = blockIdx.x;
    int64_t lo, hi;
    block_range(blocks[b], first, end_u, lo, hi);
    const int64_t e = entry[b], m = e < 0 ? hi : merge[b];
    for (int64_t o = lo + lane; o < m; o += 32) mark[o] = 0;
    __syncwarp();
    if (lane == 0 && e >= 0)
        for (int64_t o = e; o < m;) {
            if (o + 4 > end_u) break;
            const int32_t bs = (int32_t)rd32(U, o);
            if (bs < 32) break;
            mark[o] = 1;
            o += 4 + (int64_t)bs;
        }
    __syncwarp();
    int n = 0;
    for (int64_t base = lo; base < hi; base += 32) n += __popc(__ballot_sync(0xffffffffu, base + lane < hi && mark[base + lane]));
    if (lane == 0) count[b] = n;
}

struct Filter {
    int32_t tid;
    int64_t start, end;
};

// read_bam's stop conditions: a later contig, or pos >= end on the wanted one
__device__ __forceinline__ bool stops(const uint8_t *U, int64_t o, const Filter &F) {
    const int32_t ref = (int32_t)rd32(U, o + 4), pos = (int32_t)rd32(U, o + 8);
    return ref > F.tid || (ref == F.tid && (int64_t)pos >= F.end);
}

// B6
__global__ void __launch_bounds__(32) bam_offsets_kernel(const Block *__restrict__ blocks, const uint8_t *__restrict__ U,
                                                         int64_t first, int64_t end_u, const uint8_t *__restrict__ mark,
                                                         const int64_t *__restrict__ base_idx, int64_t cap,
                                                         int64_t *__restrict__ rec_off, Filter F, unsigned long long *stop) {
    const int lane = threadIdx.x, b = blockIdx.x;
    int64_t lo, hi;
    block_range(blocks[b], first, end_u, lo, hi);
    int64_t k = base_idx[b];
    for (int64_t base = lo; base < hi; base += 32) {
        const int64_t o = base + lane;
        const bool m = o < hi && mark[o];
        const unsigned bal = __ballot_sync(0xffffffffu, m);
        if (m) {
            const int64_t i = k + __popc(bal & ((1u << lane) - 1));
            if (i < cap) {
                rec_off[i] = o;
                if (o + REC_MIN <= end_u && stops(U, o, F)) atomicMin(stop, (unsigned long long)i);
            }
        }
        k += __popc(bal);
    }
}

struct ParseArgs {
    const uint8_t *U;
    int64_t end_u;
    const int64_t *rec_off;
    const int64_t *n_rec;                       // device: records
    const unsigned long long *stop;             // device: the first record that ends the run
    unsigned long long *err;                    // device: (record << 4 | error) of the first malformed record
    Filter F;
    int fa_fields;
    int32_t *keep, *n_cig, *n_seq, *n_qual, *n_name, *n_mv;   // [records + 1], 0 for a record not kept
    int64_t *mv_at;                             // first byte of the kept record's mv values
    uint8_t *mv_type;                           // their B subtype
    int64_t *cig_src;                           // first byte of the kept record's CIGAR: inline, or its CG tag's words
};

__device__ __forceinline__ int aux_size(uint8_t t) {
    switch (t) {
        case 'A': case 'c': case 'C': return 1;
        case 's': case 'S': return 2;
        case 'i': case 'I': case 'f': return 4;
        default: return 0;
    }
}

// B7
__global__ void bam_parse_kernel(ParseArgs A) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, n = *A.n_rec;
    if (i > n) return;
    int32_t keep = 0, nc = 0, ns = 0, nq = 0, nn = 0, nm = 0;
    const unsigned long long stop = *A.stop;
    if (i < n && (unsigned long long)i <= stop) {
        const uint8_t *U = A.U;
        const int64_t o = A.rec_off[i];
        const int32_t bs = (int32_t)rd32(U, o);
        const int64_t need = o + REC_MIN <= A.end_u ? fields_bytes(U, o) : -1;
        if (need < 0 || bs < need || o + 4 + (int64_t)bs > A.end_u) {
            atomicMin(A.err, (unsigned long long)i << 4 | REC_FIELDS);
        } else if ((unsigned long long)i < stop && (int32_t)rd32(U, o + 4) == A.F.tid) {
            const int32_t pos = (int32_t)rd32(U, o + 8);
            const int l_name = U[o + 12];
            const int32_t l_seq = (int32_t)rd32(U, o + 20);
            int64_t c0 = o + 36 + l_name;
            int n_cig = (int)rd16(U, o + 16);
            ns = (l_seq + 1) / 2;
            // the aux walk: read_bam's _aux_mv with fa_fields (the first "mv" B-array of an integer subtype, widened to int32),
            // and the first CG tag of a record whose CIGAR is the placeholder <l_seq>S<ref_len>N (read_bam's _cg_cigar)
            bool want_mv = A.fa_fields != 0;
            bool want_cg = false;
            if (n_cig > 0 && pos >= 0) {
                const uint32_t w0 = rd32(U, c0);
                want_cg = (w0 & 15) == 4 && w0 >> 4 == (uint32_t)l_seq;
            }
            int64_t p = c0 + 4ll * n_cig + ns + l_seq;
            const int64_t e = o + 4 + (int64_t)bs;
            bool bad = false;
            while ((want_mv || want_cg) && p + 3 <= e) {
                const uint8_t t = U[p + 2];
                const bool cg = U[p] == 'C' && U[p + 1] == 'G';
                if (want_cg && cg) {                        // only the first CG tag counts, whatever its type
                    want_cg = false;
                    if (t == 'B' && p + 8 <= e && (U[p + 3] == 'I' || U[p + 3] == 'i')) {
                        const uint32_t cnt = rd32(U, p + 4);
                        if (cnt >= (uint32_t)n_cig && cnt < CG_MAX && p + 8 + 4ll * cnt <= e) {
                            c0 = p + 8;
                            n_cig = (int)cnt;
                        }
                    }
                }
                if (t == 'B') {
                    if (p + 8 > e) { bad = true; break; }
                    const uint8_t sub = U[p + 3];
                    const int32_t cnt = (int32_t)rd32(U, p + 4);
                    const int sz = aux_size(sub) ? aux_size(sub) : 4;
                    if (cnt < 0 || p + 8 + (int64_t)cnt * sz > e) { bad = true; break; }
                    if (want_mv && U[p] == 'm' && U[p + 1] == 'v' && sub != 'A' && sub != 'f' && aux_size(sub)) {
                        nm = cnt;
                        A.mv_at[i] = p + 8;
                        A.mv_type[i] = sub;
                        want_mv = false;
                    }
                    p += 8 + (int64_t)cnt * sz;
                } else if (t == 'Z' || t == 'H') {
                    int64_t z = p + 3;
                    while (z < e && U[z]) ++z;
                    if (z >= e) { bad = true; break; }
                    p = z + 1;
                } else if (aux_size(t)) {
                    p += 3 + aux_size(t);
                } else {
                    bad = true;
                    break;
                }
            }
            int64_t span = 0;
            for (int j = 0; j < n_cig; ++j) {
                const uint32_t w = rd32(U, c0 + 4ll * j), op = w & 15;
                if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) span += w >> 4;
            }
            keep = (int64_t)pos + (span > 1 ? span : 1) > A.F.start;
            // malformed aux fields are an error only where read_bam's mv walk meets them: in a kept record, before its mv
            if (keep && bad && want_mv) {
                atomicMin(A.err, (unsigned long long)i << 4 | REC_AUX);
                keep = 0;
            }
            if (keep) {
                nc = n_cig;
                A.cig_src[i] = c0;
                if (A.fa_fields) { nq = l_seq; nn = l_name - 1; }
            } else {
                ns = nm = 0;
            }
        }
    }
    A.keep[i] = keep; A.n_cig[i] = nc; A.n_seq[i] = ns;
    if (A.fa_fields) { A.n_qual[i] = nq; A.n_name[i] = nn; A.n_mv[i] = nm; }
}

struct ScatterArgs {
    const uint8_t *U;
    const int64_t *rec_off, *n_rec;
    const int32_t *keep, *n_mv;
    const int64_t *kidx, *cig_at, *seq_at, *qual_at, *name_at, *mv_at_out;   // exclusive scans: where each record goes
    const int64_t *mv_at, *cig_src;
    const uint8_t *mv_type;
    int fa_fields;
    // outputs
    int64_t *pos;
    uint16_t *flag;
    uint8_t *mapq;
    int32_t *l_qseq;
    int64_t *cigar_off, *seq_off, *qual_off, *qname_off, *mv_off;
    uint32_t *cigar;
    uint8_t *seq, *qual, *qname;
    int32_t *mv;
};

// B9
__global__ void __launch_bounds__(WARPS * 32) bam_scatter_kernel(ScatterArgs A) {
    const int lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * WARPS + (threadIdx.x >> 5), n = *A.n_rec;
    if (i > n) return;
    const int64_t k = A.kidx[i];
    if (i == n) {                               // the closing offsets
        if (lane == 0) {
            A.cigar_off[k] = A.cig_at[i]; A.seq_off[k] = A.seq_at[i];
            if (A.fa_fields) { A.qual_off[k] = A.qual_at[i]; A.qname_off[k] = A.name_at[i]; A.mv_off[k] = A.mv_at_out[i]; }
        }
        return;
    }
    if (!A.keep[i]) return;
    const uint8_t *U = A.U;
    const int64_t o = A.rec_off[i];
    const int l_name = U[o + 12];
    const int32_t l_seq = (int32_t)rd32(U, o + 20);
    const int64_t s0 = o + 36 + l_name + 4ll * rd16(U, o + 16), ns = (l_seq + 1) / 2, q0 = s0 + ns;
    const int64_t ca = A.cig_at[i], sa = A.seq_at[i], c0 = A.cig_src[i], n_cig = A.cig_at[i + 1] - ca;
    if (lane == 0) {
        A.pos[k] = (int32_t)rd32(U, o + 8);
        A.mapq[k] = U[o + 13];
        A.flag[k] = (uint16_t)rd16(U, o + 18);
        A.l_qseq[k] = l_seq;
        A.cigar_off[k] = ca; A.seq_off[k] = sa;
    }
    for (int64_t j = lane; j < n_cig; j += 32) A.cigar[ca + j] = rd32(U, c0 + 4 * j);
    for (int64_t j = lane; j < ns; j += 32) A.seq[sa + j] = U[s0 + j];
    if (!A.fa_fields) return;
    const int64_t qa = A.qual_at[i], na = A.name_at[i], ma = A.mv_at_out[i];
    if (lane == 0) { A.qual_off[k] = qa; A.qname_off[k] = na; A.mv_off[k] = ma; }
    for (int64_t j = lane; j < l_seq; j += 32) A.qual[qa + j] = U[q0 + j];
    for (int j = lane; j < l_name - 1; j += 32) A.qname[na + j] = U[o + 36 + j];
    const int32_t nm = A.n_mv[i];
    if (nm) {
        const int64_t p = A.mv_at[i];
        const uint8_t t = A.mv_type[i];
        for (int j = lane; j < nm; j += 32) {
            int32_t v;
            switch (t) {
                case 'c': v = (int8_t)U[p + j]; break;
                case 'C': v = U[p + j]; break;
                case 's': v = (int16_t)rd16(U, p + 2ll * j); break;
                case 'S': v = (int32_t)rd16(U, p + 2ll * j); break;
                default: v = (int32_t)rd32(U, p + 4ll * j); break;     // 'i', and 'I' as numpy's astype(int32) wraps it
            }
            A.mv[ma + j] = v;
        }
    }
}

// c3b_fasta_fetch's gather, after bam_inflate has inflated the window's blocks: one thread per base of the window.  Base i sits (r + i) / lb lines and (r + i) % lb bases past the
// start of the line that holds the window's first base, which lies r bases before u0; the line ends between are skipped.
__global__ void fasta_gather_kernel(const uint8_t *__restrict__ U, int64_t u0, int64_t r, int64_t lb, int64_t lw, int64_t n,
                                    uint8_t *__restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t k = r + i;
    out[i] = U[u0 - r + k / lb * lw + k % lb];
}

constexpr int Z_THREADS = 128;              // warp 0: the compressor (one thread), warp 1: the CRC; all four load
constexpr int SYM_SLOT = 49152;             // a CTA's symbol buffer in global memory: deflate.cuh's SYM_END bytes, rounded up
constexpr size_t Z_TREES_AT = c3b_deflate::WINDOW + 2 * 32768 * 2;
constexpr size_t Z_CRC_AT = Z_TREES_AT + (sizeof(c3b_deflate::Trees) + 15) / 16 * 16;
constexpr size_t Z_SMEM = Z_CRC_AT + 256 * 4;

// Z1.  Shared memory: the 64 KiB window, head and prev (32 Ki uint16 each), the Huffman trees (8,104 B) and the CRC table:
// 205,744 B, so one encoder per SM.  The symbol buffer, 16,383 x 3 bytes, does not fit beside them and lives in the CTA's slot of sym.
// size[b]: the block's total bytes; 0 and a bad word (b << 4 | status) when its stream would not fit the 64 KiB block.
__global__ void __launch_bounds__(Z_THREADS) bgzf_deflate_kernel(const uint8_t *__restrict__ src, int64_t n, int nb,
                                                                 uint8_t *__restrict__ slots, int32_t *__restrict__ size,
                                                                 uint8_t *__restrict__ sym, unsigned long long *bad) {
    using namespace c3b_deflate;
    extern __shared__ __align__(16) uint8_t smem[];
    uint8_t *window = smem;
    uint16_t *head = reinterpret_cast<uint16_t *>(smem + WINDOW), *prev = head + 32768;
    Trees *trees = reinterpret_cast<Trees *>(smem + Z_TREES_AT);
    uint32_t *crc_tab = reinterpret_cast<uint32_t *>(smem + Z_CRC_AT);
    __shared__ uint32_t crc;
    __shared__ int clen;
    const int tid = threadIdx.x;
    for (int i = tid; i < 256; i += Z_THREADS) crc_tab[i] = crc_table_entry(i);
    for (int b = blockIdx.x; b < nb; b += gridDim.x) {
        const int64_t p0 = (int64_t)b * PAYLOAD;
        const int len = (int)(n - p0 < PAYLOAD ? n - p0 : PAYLOAD);
        const uint8_t *p = src + p0;
        reset_block(window, head, prev, p, len, tid, Z_THREADS);
        __syncthreads();
        uint8_t *blk = slots + (int64_t)b * BLOCK_MAX;
        if (tid == 0) {
            Deflater z;
            z.window = window;
            z.head = head;
            z.prev = prev;
            z.sym = sym + (int64_t)blockIdx.x * SYM_SLOT;
            z.t = trees;
            z.out = blk + HEADER;
            z.cap = BLOCK_MAX - HEADER - FOOTER;
            clen = z.run(len);
        } else if (tid >= 32 && tid < 64) {
            uint32_t term = crc_lane_term(crc_tab, p, len, tid - 32);
            for (int d = 16; d; d >>= 1) term ^= __shfl_xor_sync(0xffffffffu, term, d);
            if (tid == 32) crc = crc_lanes_done(term, len);
        }
        __syncthreads();
        if (tid == 0) {
            if (clen < 0) {
                size[b] = 0;
                atomicMin(bad, (unsigned long long)b << 4 | c3b_deflate::OUTPUT_OVERFLOW);
            } else {
                bgzf_header(blk, clen);
                put32(blk + HEADER + clen, crc);
                put32(blk + HEADER + clen + 4, (uint32_t)len);
                size[b] = HEADER + clen + FOOTER;
            }
        }
    }
}

// Z3
__global__ void __launch_bounds__(256) bgzf_pack_kernel(const uint8_t *__restrict__ slots, const int32_t *__restrict__ size,
                                                        const int64_t *__restrict__ off, uint8_t *__restrict__ image) {
    const int b = blockIdx.x;
    const uint8_t *s = slots + (int64_t)b * c3b_deflate::BLOCK_MAX;
    uint8_t *d = image + off[b];
    for (int i = threadIdx.x; i < size[b]; i += 256) d[i] = s[i];
}

size_t inflate_smem() { return 65536 + (sizeof(Tables) + 15) / 16 * 16 + 256 * 4; }

const char *status_name(int st) {
    switch (st) {
        case BAD_BLOCK_TYPE: return "bad DEFLATE block type";
        case BAD_STORED_LENGTH: return "stored block length does not match its complement";
        case BAD_CODE_LENGTHS: return "malformed Huffman code lengths";
        case BAD_CODE: return "invalid Huffman code";
        case BAD_DISTANCE: return "back-reference distance reaches before the block's start";
        case OUTPUT_OVERFLOW: return "inflates past its ISIZE";
        case INPUT_OVERRUN: return "DEFLATE stream runs past the block's compressed data";
        case SIZE_MISMATCH: return "inflated size differs from its ISIZE";
        case CRC_MISMATCH: return "CRC32 mismatch";
        default: return "unknown error";
    }
}

}  // namespace

// The decoder's workspace: the region workspace's device, stream, events (stage 0: the decode's kernels) and counter block, the
// upload staging, and the decode's buffers.
struct c3b_bam : C3bRegionWorkspace {
    uint8_t *staging = nullptr;                  // pinned: the block table, then the bytes
    size_t staging_cap = 0;
    cudaEvent_t uploaded = nullptr;              // the staging buffer is free again
    C3bBuf in, U, mark, spec_exit, entry, merge, bcount, bbase, rec_off;
    C3bBuf keep, c_cig, c_seq, c_qual, c_name, c_mv, mv_at, mv_type, cig_src;     // per record: kept, its counts, its CIGAR
    C3bBuf kidx, cig_at, seq_at, qual_at, name_at, mvo_at;
    C3bBuf pos, flag, mapq, lq, cig_off, seq_off, qual_off, name_off, mv_off, cigar, seq, qual, name, mv;
    std::vector<Block> blocks;
    std::vector<int64_t> block_start;            // offset of each block in the caller's bytes, for the errors
    int64_t n_bytes = 0;
    bool decoded = false, sized = false, fa_fields = false;
    int64_t n_reads = 0, n_cigar_out = 0, n_seq_out = 0, n_qual = 0, n_name = 0, n_mv_out = 0;   // totals
    // the last FASTA fetch: its bad-block word on the device and its pinned copy, the event after that copy, and the offsets of
    // its blocks for the error
    C3bBuf fasta_bad;
    unsigned long long *fasta_bad_host = nullptr;
    cudaEvent_t fetched = nullptr;
    std::vector<int64_t> fasta_block_start;
    bool fasta_pending = false, timed = false;
    // the last BGZF write: its slots, sizes, symbol buffers and file image; on the device its bad word, file size and block
    // offsets, and their pinned copy; the event after that copy
    C3bBuf z_slots, z_size, z_sym, z_image, z_meta;
    int64_t *z_host = nullptr;
    size_t z_host_cap = 0;
    cudaEvent_t compressed = nullptr;
    int64_t z_blocks = 0, z_bytes = 0;
    bool z_pending = false, z_sized = false;
    ~c3b_bam() {
        if (z_host) cudaFreeHost(z_host);
        if (compressed) cudaEventDestroy(compressed);
        if (staging) cudaFreeHost(staging);
        if (uploaded) cudaEventDestroy(uploaded);
        if (fasta_bad_host) cudaFreeHost(fasta_bad_host);
        if (fetched) cudaEventDestroy(fetched);
    }
};

// Checks the BGZF block headers of bytes[0 .. n) and lists the blocks.  `who` names the entry point in the error.
static int bam_blocks(const uint8_t *p, int64_t n, std::vector<Block> &out, std::vector<int64_t> &at, int64_t *total, const char *who) {
    out.clear();
    at.clear();
    int64_t o = 0, u = 0;
    while (o < n) {
        if (n - o < 18) { c3b_set_error("%s: %lld trailing bytes at offset %lld are not a BGZF block", who, (long long)(n - o), (long long)o); return 1; }
        if (p[o] != 0x1f || p[o + 1] != 0x8b || p[o + 2] != 8 || p[o + 3] != 4) {
            c3b_set_error("%s: the block at offset %lld is not a BGZF block (gzip header %02x %02x %02x %02x, want 1f 8b 08 04)", who,
                          (long long)o, p[o], p[o + 1], p[o + 2], p[o + 3]);
            return 1;
        }
        const int xlen = p[o + 10] | p[o + 11] << 8;
        if (o + 12 + xlen > n) { c3b_set_error("%s: the extra field of the block at offset %lld runs past the data", who, (long long)o); return 1; }
        int bsize = -1;
        for (int x = 0; x + 4 <= xlen;) {
            const uint8_t *f = p + o + 12 + x;
            const int slen = f[2] | f[3] << 8;
            if (x + 4 + slen > xlen) break;
            if (f[0] == 'B' && f[1] == 'C' && slen == 2) { bsize = f[4] | f[5] << 8; break; }
            x += 4 + slen;
        }
        if (bsize < 0) { c3b_set_error("%s: the block at offset %lld has no BC subfield", who, (long long)o); return 1; }
        const int64_t len = (int64_t)bsize + 1;
        if (len < 12 + xlen + 8 || o + len > n) {
            c3b_set_error("%s: BSIZE %d of the block at offset %lld is out of range", who, bsize, (long long)o);
            return 1;
        }
        const uint8_t *foot = p + o + len - 8;
        const uint32_t crc = foot[0] | foot[1] << 8 | foot[2] << 16 | (uint32_t)foot[3] << 24;
        const uint32_t isize = foot[4] | foot[5] << 8 | foot[6] << 16 | (uint32_t)foot[7] << 24;
        if (isize > 65536) { c3b_set_error("%s: ISIZE %u of the block at offset %lld exceeds 65536", who, isize, (long long)o); return 1; }
        Block b;
        b.coff = o + 12 + xlen;
        b.uoff = u;
        b.clen = (int32_t)(len - 12 - xlen - 8);
        b.isize = (int32_t)isize;
        b.crc = crc;
        b.pad = 0;
        out.push_back(b);
        at.push_back(o);
        u += isize;
        o += len;
    }
    *total = u;
    return 0;
}

// Waits until the previous upload has left the pinned staging buffer, and grows it to hold up bytes.
static int bam_staging(c3b_bam *w, size_t up, const char *who) {
    C3B_CUDA(cudaEventSynchronize(w->uploaded));
    if (up > w->staging_cap) {
        if (w->staging) cudaFreeHost(w->staging);
        w->staging = nullptr;
        w->staging_cap = 0;
        const size_t want = up + up / 4 + 4096;
        if (cudaMallocHost((void **)&w->staging, want) != cudaSuccess) { c3b_set_error("%s: pinned allocation of %zu bytes failed", who, want); return 1; }
        w->staging_cap = want;
    }
    return 0;
}

// Copies the block table (w->blocks) and bytes[0 .. n_bytes) into the pinned staging buffer.  bam_upload then queues the
// staged bytes into w->in.
static int bam_stage(c3b_bam *w, const uint8_t *bytes, int64_t n_bytes, const char *who) {
    const size_t table = w->blocks.size() * sizeof(Block), up = table + (size_t)n_bytes;
    if (bam_staging(w, up, who)) return 1;
    if (table) memcpy(w->staging, w->blocks.data(), table);
    if (n_bytes) memcpy(w->staging + table, bytes, (size_t)n_bytes);
    return 0;
}

static int bam_upload(c3b_bam *w, size_t up, cudaStream_t s) {
    if (up) C3B_CUDA(cudaMemcpyAsync(w->in.p, w->staging, up, cudaMemcpyHostToDevice, s));
    C3B_CUDA(cudaEventRecord(w->uploaded, s));
    return 0;
}

static inline unsigned bam_grid(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }

extern "C" {

int c3b_bam_create(c3b_bam **out, int device_ordinal) {
    if (c3b_region_create(out, device_ordinal, 1, N_COUNTERS, 0, "c3b_bam_create")) return 1;
    c3b_bam *w = *out;
    if (cudaEventCreateWithFlags(&w->uploaded, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&w->fetched, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&w->compressed, cudaEventDisableTiming) != cudaSuccess ||
        cudaMallocHost((void **)&w->fasta_bad_host, 8) != cudaSuccess || w->fasta_bad.ensure(8, nullptr, "c3b_bam_create") ||
        cudaFuncSetAttribute(bam_inflate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)inflate_smem()) != cudaSuccess ||
        cudaFuncSetAttribute(bgzf_deflate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Z_SMEM) != cudaSuccess) {
        c3b_set_error("c3b_bam_create: event creation, a small allocation or a kernel's shared-memory setting failed");
        c3b_bam_destroy(w);
        *out = nullptr;
        return 1;
    }
    return 0;
}

int c3b_bam_decode(c3b_bam *w, const uint8_t *bytes, int64_t n_bytes, int64_t first_uoff, int64_t end_uoff, int32_t tid,
                   int64_t start, int64_t end, int fa_fields, void *cuda_stream) {
    const char *who = "c3b_bam_decode";
    if (!w || (n_bytes > 0 && !bytes) || n_bytes < 0) { c3b_set_error("%s: null argument", who); return 1; }
    if (tid < 0) { c3b_set_error("%s: tid %d < 0", who, tid); return 1; }
    w->decoded = w->sized = false;
    int64_t total = 0;
    if (bam_blocks(bytes, n_bytes, w->blocks, w->block_start, &total, who)) return 1;
    if (end_uoff == -1) end_uoff = total;
    if (first_uoff < 0 || end_uoff < first_uoff || end_uoff > total) {
        c3b_set_error("%s: first_uoff %lld / end_uoff %lld outside the %lld uncompressed bytes", who, (long long)first_uoff,
                      (long long)end_uoff, (long long)total);
        return 1;
    }
    C3B_CUDA(cudaSetDevice(w->device));
    cudaStream_t s = (cudaStream_t)cuda_stream;
    w->stream = s;
    w->fa_fields = fa_fields != 0;
    w->n_bytes = n_bytes;
    const int nb = (int)w->blocks.size();
    const size_t table = (size_t)nb * sizeof(Block);
    if (bam_stage(w, bytes, n_bytes, who)) return 1;

    const int64_t Uz = total > 0 ? total : 1, cap = total / REC_MIN + 1, nbz = nb > 0 ? nb : 1;
    auto grow = [&](C3bBuf &b, size_t bytes_) { return b.ensure(bytes_ ? bytes_ : 1, s, "c3b_bam"); };
    const size_t c1 = (size_t)cap + 1;
    if (grow(w->in, table + (size_t)n_bytes) || grow(w->U, (size_t)Uz) || grow(w->mark, (size_t)Uz) || grow(w->spec_exit, nbz * 8) ||
        grow(w->entry, nbz * 8) || grow(w->merge, nbz * 8) || grow(w->bcount, (nbz + 1) * 4) || grow(w->bbase, (nbz + 1) * 8) ||
        grow(w->rec_off, (size_t)cap * 8) || grow(w->keep, c1 * 4) || grow(w->c_cig, c1 * 4) || grow(w->c_seq, c1 * 4) ||
        grow(w->kidx, c1 * 8) || grow(w->cig_src, c1 * 8) || grow(w->cig_at, c1 * 8) || grow(w->seq_at, c1 * 8) || grow(w->pos, (size_t)cap * 8) ||
        grow(w->flag, (size_t)cap * 2) || grow(w->mapq, (size_t)cap) || grow(w->lq, (size_t)cap * 4) || grow(w->cig_off, c1 * 8) ||
        grow(w->seq_off, c1 * 8) || grow(w->cigar, (size_t)Uz) || grow(w->seq, (size_t)Uz))
        return 1;
    if (w->fa_fields &&
        (grow(w->c_qual, c1 * 4) || grow(w->c_name, c1 * 4) || grow(w->c_mv, c1 * 4) || grow(w->mv_at, c1 * 8) ||
         grow(w->mv_type, c1) || grow(w->qual_at, c1 * 8) || grow(w->name_at, c1 * 8) || grow(w->mvo_at, c1 * 8) ||
         grow(w->qual_off, c1 * 8) || grow(w->name_off, c1 * 8) || grow(w->mv_off, c1 * 8) || grow(w->qual, (size_t)Uz) ||
         grow(w->name, (size_t)Uz) || grow(w->mv, (size_t)Uz * 4)))
        return 1;
    if (bam_upload(w, table + (size_t)n_bytes, s)) return 1;

    int64_t *cnt = w->counters.as<int64_t>();
    unsigned long long *bad = reinterpret_cast<unsigned long long *>(cnt), *stop = bad + 1, *err = bad + 2;
    C3B_CUDA(cudaMemsetAsync(cnt, 0xff, 3 * 8, s));
    C3B_CUDA(cudaMemsetAsync(cnt + 3, 0, (N_COUNTERS - 3) * 8, s));
    const Block *B = w->in.as<Block>();
    const uint8_t *bytes_d = w->in.as<uint8_t>() + table;
    uint8_t *U = w->U.as<uint8_t>();
    w->launches[0] = 0;
    C3B_CUDA(cudaEventRecord(w->ev[0][0], s));
    if (nb > 0) {
        const Filter F{tid, start, end};
        C3B_CUDA(cudaMemsetAsync(w->mark.p, 0, (size_t)Uz, s));
        bam_inflate_kernel<<<nb, 32, inflate_smem(), s>>>(bytes_d, B, U, bad);
        bam_speculate_kernel<<<nb, 32, 0, s>>>(B, U, first_uoff, end_uoff, w->mark.as<uint8_t>(), w->spec_exit.as<int64_t>());
        bam_fixup_kernel<<<1, 1, 0, s>>>(B, nb, U, first_uoff, end_uoff, w->mark.as<uint8_t>(), w->spec_exit.as<int64_t>(),
                                         w->entry.as<int64_t>(), w->merge.as<int64_t>(), cnt);
        bam_starts_kernel<<<nb, 32, 0, s>>>(B, U, first_uoff, end_uoff, w->mark.as<uint8_t>(), w->entry.as<int64_t>(),
                                            w->merge.as<int64_t>(), w->bcount.as<int32_t>());
        block_scan_sum(w->bcount.as<int32_t>(), w->bbase.as<int64_t>(), nb, nullptr, cnt + 5, s);
        bam_offsets_kernel<<<nb, 32, 0, s>>>(B, U, first_uoff, end_uoff, w->mark.as<uint8_t>(), w->bbase.as<int64_t>(), cap,
                                             w->rec_off.as<int64_t>(), F, stop);
        ParseArgs P;
        P.U = U; P.end_u = end_uoff; P.rec_off = w->rec_off.as<int64_t>(); P.n_rec = cnt + 5; P.stop = stop; P.err = err; P.F = F;
        P.fa_fields = w->fa_fields;
        P.keep = w->keep.as<int32_t>(); P.n_cig = w->c_cig.as<int32_t>(); P.n_seq = w->c_seq.as<int32_t>();
        P.n_qual = w->c_qual.as<int32_t>(); P.n_name = w->c_name.as<int32_t>(); P.n_mv = w->c_mv.as<int32_t>();
        P.mv_at = w->mv_at.as<int64_t>(); P.mv_type = w->mv_type.as<uint8_t>(); P.cig_src = w->cig_src.as<int64_t>();
        bam_parse_kernel<<<bam_grid(cap + 1, 256), 256, 0, s>>>(P);
        // record counts: the scans read records + 1 entries (the last is 0) and leave the totals in the counter block
        block_scan_sum(w->keep.as<int32_t>(), w->kidx.as<int64_t>(), cap + 1, cnt + 5, cnt + 6, s);
        block_scan_sum(w->c_cig.as<int32_t>(), w->cig_at.as<int64_t>(), cap + 1, cnt + 5, cnt + 7, s);
        block_scan_sum(w->c_seq.as<int32_t>(), w->seq_at.as<int64_t>(), cap + 1, cnt + 5, cnt + 8, s);
        w->launches[0] += 10;
        if (w->fa_fields) {
            block_scan_sum(w->c_qual.as<int32_t>(), w->qual_at.as<int64_t>(), cap + 1, cnt + 5, cnt + 9, s);
            block_scan_sum(w->c_name.as<int32_t>(), w->name_at.as<int64_t>(), cap + 1, cnt + 5, cnt + 10, s);
            block_scan_sum(w->c_mv.as<int32_t>(), w->mvo_at.as<int64_t>(), cap + 1, cnt + 5, cnt + 11, s);
            w->launches[0] += 3;
        }
        ScatterArgs S;
        S.U = U; S.rec_off = w->rec_off.as<int64_t>(); S.n_rec = cnt + 5; S.keep = w->keep.as<int32_t>(); S.n_mv = w->c_mv.as<int32_t>();
        S.kidx = w->kidx.as<int64_t>(); S.cig_at = w->cig_at.as<int64_t>(); S.seq_at = w->seq_at.as<int64_t>();
        S.qual_at = w->qual_at.as<int64_t>(); S.name_at = w->name_at.as<int64_t>(); S.mv_at_out = w->mvo_at.as<int64_t>();
        S.mv_at = w->mv_at.as<int64_t>(); S.cig_src = w->cig_src.as<int64_t>(); S.mv_type = w->mv_type.as<uint8_t>(); S.fa_fields = w->fa_fields;
        S.pos = w->pos.as<int64_t>(); S.flag = w->flag.as<uint16_t>(); S.mapq = w->mapq.as<uint8_t>(); S.l_qseq = w->lq.as<int32_t>();
        S.cigar_off = w->cig_off.as<int64_t>(); S.seq_off = w->seq_off.as<int64_t>(); S.qual_off = w->qual_off.as<int64_t>();
        S.qname_off = w->name_off.as<int64_t>(); S.mv_off = w->mv_off.as<int64_t>();
        S.cigar = w->cigar.as<uint32_t>(); S.seq = w->seq.as<uint8_t>(); S.qual = w->qual.as<uint8_t>(); S.qname = w->name.as<uint8_t>();
        S.mv = w->mv.as<int32_t>();
        bam_scatter_kernel<<<bam_grid(cap + 1, WARPS), WARPS * 32, 0, s>>>(S);
        w->launches[0] += 1;
    } else {
        // no blocks: no records; the closing offsets are the only output
        for (C3bBuf *b : {&w->cig_off, &w->seq_off, &w->qual_off, &w->name_off, &w->mv_off})
            if (b->p) C3B_CUDA(cudaMemsetAsync(b->p, 0, 8, s));
    }
    C3B_CUDA(cudaEventRecord(w->ev[0][1], s));
    C3B_CUDA(cudaGetLastError());
    C3B_CUDA(cudaMemcpyAsync(w->host_counters, cnt, N_COUNTERS * 8, cudaMemcpyDeviceToHost, s));
    w->decoded = w->timed = true;
    return 0;
}

int c3b_fasta_fetch(c3b_bam *w, const uint8_t *bytes, int64_t n_bytes, int64_t first_uoff, int64_t start, int64_t line_bases,
                    int64_t line_bytes, int64_t n_bases, uint8_t *out, void *cuda_stream) {
    const char *who = "c3b_fasta_fetch";
    if (!w || (n_bytes > 0 && !bytes) || n_bytes < 0 || n_bases < 0 || (n_bases > 0 && !out)) {
        c3b_set_error("%s: null or negative argument", who);
        return 1;
    }
    w->fasta_pending = false;
    if (n_bases == 0) return 0;
    if (line_bases <= 0 || line_bytes < line_bases || start < 0 || first_uoff < 0) {
        c3b_set_error("%s: line bases %lld / line bytes %lld / start %lld / first_uoff %lld are not a FASTA window's", who,
                      (long long)line_bases, (long long)line_bytes, (long long)start, (long long)first_uoff);
        return 1;
    }
    int64_t total = 0;
    if (bam_blocks(bytes, n_bytes, w->blocks, w->fasta_block_start, &total, who)) return 1;
    const int64_t r = start % line_bases, k = r + n_bases - 1;
    const int64_t last = first_uoff - r + k / line_bases * line_bytes + k % line_bases;
    if (last >= total) {
        c3b_set_error("%s: the window's last base at uncompressed offset %lld lies past the %lld bytes its blocks inflate to", who,
                      (long long)last, (long long)total);
        return 1;
    }
    C3B_CUDA(cudaSetDevice(w->device));
    cudaStream_t s = (cudaStream_t)cuda_stream;
    w->stream = s;
    const int nb = (int)w->blocks.size();
    const size_t table = (size_t)nb * sizeof(Block);
    if (bam_stage(w, bytes, n_bytes, who)) return 1;
    if (w->in.ensure(table + (size_t)n_bytes, s, "c3b_bam") || w->U.ensure((size_t)total, s, "c3b_bam")) return 1;
    if (bam_upload(w, table + (size_t)n_bytes, s)) return 1;
    unsigned long long *bad = w->fasta_bad.as<unsigned long long>();
    C3B_CUDA(cudaMemsetAsync(bad, 0xff, 8, s));
    C3B_CUDA(cudaEventRecord(w->ev[0][0], s));
    bam_inflate_kernel<<<nb, 32, inflate_smem(), s>>>(w->in.as<uint8_t>() + table, w->in.as<Block>(), w->U.as<uint8_t>(), bad);
    fasta_gather_kernel<<<bam_grid(n_bases, 256), 256, 0, s>>>(w->U.as<uint8_t>(), first_uoff, r, line_bases, line_bytes, n_bases, out);
    C3B_CUDA(cudaEventRecord(w->ev[0][1], s));
    C3B_CUDA(cudaGetLastError());
    w->launches[0] = 2;
    w->timed = true;
    C3B_CUDA(cudaMemcpyAsync(w->fasta_bad_host, bad, 8, cudaMemcpyDeviceToHost, s));
    C3B_CUDA(cudaEventRecord(w->fetched, s));
    w->fasta_pending = true;
    return 0;
}

int c3b_fasta_status(c3b_bam *w) {
    const char *who = "c3b_fasta_status";
    if (!w) { c3b_set_error("%s: null argument", who); return 1; }
    if (!w->fasta_pending) return 0;
    C3B_CUDA(cudaSetDevice(w->device));
    C3B_CUDA(cudaEventSynchronize(w->fetched));
    w->fasta_pending = false;
    const unsigned long long bad = *w->fasta_bad_host;
    if (bad != ~0ull) {
        const size_t b = (size_t)(bad >> 4);
        c3b_set_error("%s: BGZF block %zu (at byte %lld of the data): %s", who, b, (long long)w->fasta_block_start[b],
                      status_name((int)(bad & 15)));
        return 1;
    }
    return 0;
}

int c3b_bam_sizes(c3b_bam *w, int64_t *n_reads, int64_t *n_cigar, int64_t *n_seq, int64_t *n_qual, int64_t *n_qname,
                  int64_t *n_mv) {
    const char *who = "c3b_bam_sizes";
    if (!w || !w->decoded) { c3b_set_error("%s: no c3b_bam_decode has been issued", who); return 1; }
    C3B_CUDA(cudaSetDevice(w->device));
    C3B_CUDA(cudaStreamSynchronize(w->stream));
    const int64_t *h = w->host_counters;
    const unsigned long long bad = (unsigned long long)h[0], stop = (unsigned long long)h[1], err = (unsigned long long)h[2];
    if (bad != ~0ull) {
        const size_t b = (size_t)(bad >> 4);
        c3b_set_error("%s: BGZF block %zu (at byte %lld of the data): %s", who, b, (long long)w->block_start[b], status_name((int)(bad & 15)));
        return 1;
    }
    if (h[3] == CHAIN_SHORT_BLOCK_SIZE) {
        c3b_set_error("%s: the record at uncompressed offset %lld has a block_size below the 32 bytes of its core fields", who,
                      (long long)h[4]);
        return 1;
    }
    if (h[3] == CHAIN_TRUNCATED) {
        c3b_set_error("%s: truncated record: the record chain reaches uncompressed offset %lld, not the end of the records", who,
                      (long long)h[4]);
        return 1;
    }
    const unsigned long long n_rec = (unsigned long long)h[5];
    if (err != ~0ull && (err >> 4) <= (stop < n_rec ? stop : n_rec)) {
        c3b_set_error("%s: record %llu of the data: %s", who, err >> 4,
                      (err & 15) == REC_AUX ? "an auxiliary field is malformed or runs past the record"
                                            : "its block_size cannot hold the fields its header declares");
        return 1;
    }
    w->n_reads = h[6]; w->n_cigar_out = h[7]; w->n_seq_out = h[8];
    w->n_qual = w->fa_fields ? h[9] : 0; w->n_name = w->fa_fields ? h[10] : 0; w->n_mv_out = w->fa_fields ? h[11] : 0;
    w->sized = true;
    if (n_reads) *n_reads = w->n_reads;
    if (n_cigar) *n_cigar = w->n_cigar_out;
    if (n_seq) *n_seq = w->n_seq_out;
    if (n_qual) *n_qual = w->n_qual;
    if (n_qname) *n_qname = w->n_name;
    if (n_mv) *n_mv = w->n_mv_out;
    return 0;
}

int c3b_bam_fetch(c3b_bam *w, const c3b_bam_out *out, int on_device) {
    const char *who = "c3b_bam_fetch";
    if (!w || !out) { c3b_set_error("%s: null argument", who); return 1; }
    if (!w->sized) { c3b_set_error("%s: call c3b_bam_sizes after c3b_bam_decode first", who); return 1; }
    if (!w->fa_fields && (out->qual_off || out->qual || out->qname_off || out->qname || out->mv_off || out->mv)) {
        c3b_set_error("%s: qualities, names and mv need a decode with fa_fields = 1", who);
        return 1;
    }
    C3B_CUDA(cudaSetDevice(w->device));
    const cudaMemcpyKind kind = on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    const size_t n = (size_t)w->n_reads, n1 = (n + 1) * 8;
    auto put = [&](void *dst, const C3bBuf &src, size_t bytes) -> int {
        if (dst && bytes) C3B_CUDA(cudaMemcpyAsync(dst, src.p, bytes, kind, w->stream));
        return 0;
    };
    if (put(out->pos, w->pos, n * 8) || put(out->flag, w->flag, n * 2) || put(out->mapq, w->mapq, n) || put(out->l_qseq, w->lq, n * 4) ||
        put(out->cigar_off, w->cig_off, n1) || put(out->cigar, w->cigar, (size_t)w->n_cigar_out * 4) ||
        put(out->seq_off, w->seq_off, n1) || put(out->seq, w->seq, (size_t)w->n_seq_out))
        return 1;
    if (w->fa_fields && (put(out->qual_off, w->qual_off, n1) || put(out->qual, w->qual, (size_t)w->n_qual) ||
                         put(out->qname_off, w->name_off, n1) || put(out->qname, w->name, (size_t)w->n_name) ||
                         put(out->mv_off, w->mv_off, n1) || put(out->mv, w->mv, (size_t)w->n_mv_out * 4)))
        return 1;
    return on_device ? 0 : w->wait();
}

int c3b_bgzf_compress(c3b_bam *w, const uint8_t *src, int64_t n, int on_device, void *cuda_stream) {
    const char *who = "c3b_bgzf_compress";
    if (!w || (n > 0 && !src) || n < 0) { c3b_set_error("%s: null or negative argument", who); return 1; }
    w->z_pending = w->z_sized = false;
    C3B_CUDA(cudaSetDevice(w->device));
    cudaStream_t s = (cudaStream_t)cuda_stream;
    w->stream = s;
    const int64_t nb = (n + c3b_deflate::PAYLOAD - 1) / c3b_deflate::PAYLOAD;
    if (nb > INT_MAX) { c3b_set_error("%s: %lld bytes are more BGZF blocks than one call takes", who, (long long)n); return 1; }
    int sms = 0;
    C3B_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, w->device));
    const int grid = (int)(nb < sms ? nb : sms);
    const size_t meta = (size_t)(nb + 2) * 8, slots = (size_t)nb * c3b_deflate::BLOCK_MAX;
    if (w->z_slots.ensure(slots ? slots : 1, s, "c3b_bam") || w->z_image.ensure(slots ? slots : 1, s, "c3b_bam") ||
        w->z_size.ensure((size_t)(nb ? nb : 1) * 4, s, "c3b_bam") || w->z_sym.ensure((size_t)(grid ? grid : 1) * SYM_SLOT, s, "c3b_bam") ||
        w->z_meta.ensure(meta, s, "c3b_bam"))
        return 1;
    if (meta > w->z_host_cap) {
        C3B_CUDA(cudaEventSynchronize(w->compressed));
        if (w->z_host) cudaFreeHost(w->z_host);
        w->z_host = nullptr;
        w->z_host_cap = 0;
        if (cudaMallocHost((void **)&w->z_host, meta) != cudaSuccess) { c3b_set_error("%s: pinned allocation of %zu bytes failed", who, meta); return 1; }
        w->z_host_cap = meta;
    }
    const uint8_t *d_src = src;
    if (!on_device && n > 0) {
        if (bam_staging(w, (size_t)n, who) || w->in.ensure((size_t)n, s, "c3b_bam")) return 1;
        memcpy(w->staging, src, (size_t)n);
        if (bam_upload(w, (size_t)n, s)) return 1;
        d_src = w->in.as<uint8_t>();
    }
    int64_t *m = w->z_meta.as<int64_t>();
    C3B_CUDA(cudaMemsetAsync(m, 0xff, 8, s));
    C3B_CUDA(cudaMemsetAsync(m + 1, 0, 8, s));
    C3B_CUDA(cudaEventRecord(w->ev[0][0], s));
    w->launches[0] = 0;
    if (nb > 0) {
        bgzf_deflate_kernel<<<grid, Z_THREADS, Z_SMEM, s>>>(d_src, n, (int)nb, w->z_slots.as<uint8_t>(), w->z_size.as<int32_t>(),
                                                           w->z_sym.as<uint8_t>(), reinterpret_cast<unsigned long long *>(m));
        block_scan_sum(w->z_size.as<int32_t>(), m + 2, nb, nullptr, m + 1, s);
        bgzf_pack_kernel<<<(unsigned)nb, 256, 0, s>>>(w->z_slots.as<uint8_t>(), w->z_size.as<int32_t>(), m + 2, w->z_image.as<uint8_t>());
        w->launches[0] = 3;
    }
    C3B_CUDA(cudaEventRecord(w->ev[0][1], s));
    C3B_CUDA(cudaGetLastError());
    C3B_CUDA(cudaMemcpyAsync(w->z_host, m, meta, cudaMemcpyDeviceToHost, s));
    C3B_CUDA(cudaEventRecord(w->compressed, s));
    w->z_blocks = nb;
    w->z_pending = w->timed = true;
    return 0;
}

int c3b_bgzf_sizes(c3b_bam *w, int64_t *n_out, int64_t *block_off) {
    const char *who = "c3b_bgzf_sizes";
    if (!w || !w->z_pending) { c3b_set_error("%s: no c3b_bgzf_compress has been issued", who); return 1; }
    C3B_CUDA(cudaSetDevice(w->device));
    C3B_CUDA(cudaEventSynchronize(w->compressed));
    const int64_t *h = w->z_host;
    const unsigned long long bad = (unsigned long long)h[0];
    if (bad != ~0ull) {
        c3b_set_error("%s: BGZF block %llu's DEFLATE stream does not fit a 64 KiB block", who, bad >> 4);
        return 1;
    }
    w->z_bytes = h[1];
    w->z_sized = true;
    if (n_out) *n_out = w->z_bytes;
    if (block_off) {
        if (w->z_blocks) memcpy(block_off, h + 2, (size_t)w->z_blocks * 8);
        block_off[w->z_blocks] = w->z_bytes;
    }
    return 0;
}

int c3b_bgzf_fetch(c3b_bam *w, uint8_t *out, int on_device) {
    const char *who = "c3b_bgzf_fetch";
    if (!w || (!out && w->z_bytes)) { c3b_set_error("%s: null argument", who); return 1; }
    if (!w->z_sized) { c3b_set_error("%s: call c3b_bgzf_sizes after c3b_bgzf_compress first", who); return 1; }
    C3B_CUDA(cudaSetDevice(w->device));
    if (w->z_bytes)
        C3B_CUDA(cudaMemcpyAsync(out, w->z_image.p, (size_t)w->z_bytes, on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, w->stream));
    return on_device ? 0 : w->wait();
}

int c3b_bam_last_ms(c3b_bam *w, float *ms, int *launches) {
    if (!w || !w->timed) { c3b_set_error("c3b_bam_last_ms: no c3b_bam_decode, c3b_fasta_fetch or c3b_bgzf_compress has been issued"); return 1; }
    return w->elapsed(0, ms, launches);
}

void c3b_bam_destroy(c3b_bam *w) { c3b_region_destroy(w); }

}  // extern "C"
