// phase.cu - read-based phasing on the GPU (include/clair3_b200_phase.h; DESIGN.md 5g.3).  clair3_b200/phasing.py states
// what is computed; this file computes the same integers.
//
//   phase_fragment_kernel<false>  one warp per record: the CIGAR in steps of 32 operations, a warp scan of each step's
//                                 reference and query lengths, and per aligned operation a binary search of the variant
//                                 positions it covers.  Writes each record's entry count (0 for a filtered record or one of
//                                 fewer than two entries).
//   (block_scan)                  exclusive sum of the counts: each record's first entry.
//   phase_fragment_kernel<true>   the same walk, writing (read, variant, allele, weight) at each record's offset, in order.
//
//   phase_dp_kernel               one 1024-thread CTA per block, over persistent CTAs that take the blocks largest first.
//                                 Forward: per column thread 0 updates the active reads (at most 15) and the column's shape;
//                                 the threads compute, per pattern of the shared reads, the minimum of the previous column over
//                                 the patterns of the leaving reads (the projection), then D over the 2^(k-1) states of the
//                                 column.  D of the last column of each segment of C3B_PHASE_SEGMENT columns goes to a
//                                 checkpoint.  Backtrace: per segment, last first, the segment is recomputed from its checkpoint
//                                 with each projection's argmin stored as the uint16 pattern of the leaving reads, and thread 0
//                                 walks it back.
#include <limits.h>

#include "block_scan.cuh"
#include "c3b_internal.h"
#include "../../include/clair3_b200_phase.h"

namespace {

constexpr uint16_t kFlagSkip = 0x4 | 0x100 | 0x200 | 0x400 | 0x800;
constexpr int kMinMapq = 20;
constexpr int kThreads = 1024;
constexpr int kMaxStates = 1 << (C3B_PHASE_MAX_READS - 1);

__device__ __forceinline__ int64_t lower_bound(const int64_t *a, int64_t n, int64_t x) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg(a + mid) < x) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

struct FragArgs {
    C3bReads r;
    int64_t lo, hi;
    c3b_phase_variants v;
    int64_t first, read_base;
};

// Write = false: counts[i] = entries of record i.  Write = true: the entries at offsets[i].  One warp per record.
template <bool Write>
__global__ void __launch_bounds__(256) phase_fragment_kernel(const FragArgs a, int64_t *counts, const int64_t *offsets,
                                                             int64_t *out_read, int32_t *out_var, uint8_t *out_allele,
                                                             uint8_t *out_weight, int64_t *first_out) {
    const int lane = threadIdx.x & 31;
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (!Write && i == 0 && lane == 0) *first_out = lower_bound(a.r.pos, a.r.n, a.lo);
    if (i >= a.r.n) return;
    const int64_t p = a.r.pos[i];
    bool take = p >= a.lo && p < a.hi && !(a.r.flag[i] & kFlagSkip) && a.r.mapq[i] >= kMinMapq;
    if (Write) take = take && offsets[i + 1] > offsets[i];
    if (!take) {
        if (!Write && lane == 0) counts[i] = 0;
        return;
    }
    const uint32_t *cig = a.r.cigar + a.r.cigar_off[i];
    const int64_t n_ops = a.r.cigar_off[i + 1] - a.r.cigar_off[i];
    const uint8_t *sq = a.r.seq + a.r.seq_off[i];
    const uint8_t *ql = a.r.qual + a.r.qual_off[i];
    const int lq = a.r.l_qseq[i];
    int64_t rbase = p, qbase = 0, n = 0, out = Write ? offsets[i] : 0;
    for (int64_t o0 = 0; o0 < n_ops; o0 += 32) {
        const int64_t o = o0 + lane;
        uint32_t op = 0, len = 0;
        if (o < n_ops) {
            const uint32_t w = __ldg(cig + o);
            op = w & 15;
            len = w >> 4;
        }
        const bool aligned = (op == 0 || op == 7 || op == 8) && o < n_ops;
        const int64_t rl = (o < n_ops && (aligned || op == 2 || op == 3)) ? len : 0;
        const int64_t qlen = (o < n_ops && (aligned || op == 1 || op == 4)) ? len : 0;
        int64_t rs = rl, qs = qlen;                                 // inclusive warp scans
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int64_t x = __shfl_up_sync(0xffffffffu, rs, d), y = __shfl_up_sync(0xffffffffu, qs, d);
            if (lane >= d) { rs += x; qs += y; }
        }
        const int64_t r0 = rbase + rs - rl, q0 = qbase + qs - qlen;
        // this lane's alleles, in variant order
        int cnt = 0;
        int64_t v0 = 0, v1 = 0;
        if (aligned && len) {
            v0 = lower_bound(a.v.pos, a.v.n, r0);
            v1 = lower_bound(a.v.pos, a.v.n, r0 + len);
            for (int64_t v = v0; v < v1; ++v) {
                const int b = c3b_nib_at(sq, lq, q0 + (a.v.pos[v] - r0));
                cnt += b == a.v.ref[v] || b == a.v.alt[v];
            }
        }
        int sc = cnt;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int x = __shfl_up_sync(0xffffffffu, sc, d);
            if (lane >= d) sc += x;
        }
        if (Write && cnt) {
            int64_t at = out + n + sc - cnt;
            for (int64_t v = v0; v < v1; ++v) {
                const int64_t q = q0 + (a.v.pos[v] - r0);
                const int b = c3b_nib_at(sq, lq, q);
                if (b != a.v.ref[v] && b != a.v.alt[v]) continue;
                out_read[at] = a.read_base + i - a.first;
                out_var[at] = (int32_t)v;
                out_allele[at] = b == a.v.alt[v];
                out_weight[at] = ql[q];
                ++at;
            }
        }
        n += __shfl_sync(0xffffffffu, sc, 31);
        rbase += __shfl_sync(0xffffffffu, rs, 31);
        qbase += __shfl_sync(0xffffffffu, qs, 31);
    }
    if (!Write && lane == 0) counts[i] = n >= 2 ? n : 0;
}

// ------------------------------------------------------------------------------------------------ the DP
struct ColMeta {
    uint16_t k, ns, sh, lv;        // active reads, of them active at the previous column too, shared / leaving bits there
};

// pdep: the low bits of x placed at the set bits of mask, lowest first.
__device__ __forceinline__ uint32_t deposit(uint32_t x, uint32_t mask) {
    uint32_t r = 0;
    for (uint32_t m = mask; m; m &= m - 1, x >>= 1)
        if (x & 1) r |= m & (0u - m);
    return r;
}

struct DpShared {
    uint32_t D[kMaxStates];        // D of the last column computed, by normalized state
    uint32_t Q[kMaxStates];        // the projection of the previous column, by pattern of the shared reads
    int32_t act[C3B_PHASE_MAX_READS + 1];
    uint8_t eb[C3B_PHASE_MAX_READS + 1], ea[C3B_PHASE_MAX_READS + 1], ew[C3B_PHASE_MAX_READS + 1];
    ColMeta meta;
    int ne, kprev, nxt, bad;
    unsigned long long red[32];
};

// opt1 = W1(S0) + W0(S1) of state B (bit 0 clear) from the column's entries in smem; opt2 = total - opt1.
__device__ __forceinline__ uint32_t opt1_of(const DpShared &S, uint32_t B) {
    uint32_t o = 0;
    for (int e = 0; e < S.ne; ++e) o += ((B >> S.eb[e]) ^ S.ea[e]) & 1 ? S.ew[e] : 0;
    return o;
}

// One column: the projection of D (the previous column, S.kprev reads) into Q, its argmins to arg (null: not kept), then the
// column's D.  S.meta, S.ne and the entries are set; first: the block's first column (no predecessor).
__device__ void dp_column(DpShared &S, bool first, uint16_t *arg) {
    const ColMeta m = S.meta;
    const int nq = first ? 1 : 1 << (m.ns - 1);
    if (!first) {
        const uint32_t fullp = (1u << S.kprev) - 1;
        for (int t = threadIdx.x; t < nq; t += kThreads) {
            const uint32_t base = deposit((uint32_t)t << 1, m.sh);
            uint32_t best = UINT_MAX, bl = 0, l = 0, sub = 0;
            do {
                const uint32_t full = base | sub;
                const uint32_t v = S.D[((full & 1) ? (~full & fullp) : full) >> 1];
                if (v < best) { best = v; bl = l; }
                ++l;
                sub = (sub - m.lv) & m.lv;
            } while (sub);
            S.Q[t] = best;
            if (arg) arg[t] = (uint16_t)bl;
        }
        __syncthreads();
    }
    uint32_t total = 0;
    for (int e = 0; e < S.ne; ++e) total += S.ew[e];
    const int ns_mask = nq - 1;
    for (int s = threadIdx.x; s < (1 << (m.k - 1)); s += kThreads) {
        const uint32_t o1 = opt1_of(S, (uint32_t)s << 1);
        const uint32_t c = o1 < total - o1 ? o1 : total - o1;
        S.D[s] = c + (first ? 0u : S.Q[s & ns_mask]);
    }
    __syncthreads();
}

// Thread 0: the column's entries (their bits from ebit, as the forward pass set them) into smem.
__device__ __forceinline__ void load_entries(DpShared &S, const c3b_phase_blocks &B, const uint8_t *ebit, int64_t c) {
    const int64_t e0 = B.ent_off[c];
    S.ne = (int)(B.ent_off[c + 1] - e0);
    for (int e = 0; e < S.ne; ++e) {
        S.eb[e] = ebit[e0 + e];
        S.ea[e] = B.ent_allele[e0 + e];
        S.ew[e] = B.ent_weight[e0 + e];
    }
}

__global__ void __launch_bounds__(kThreads, 1) phase_dp_kernel(const c3b_phase_blocks B, uint8_t *hap, int64_t *cost,
                                                               uint32_t *ckpt, uint16_t *seg_all, int64_t seg_stride,
                                                               uint16_t *meta_all, uint8_t *ebit, int64_t *status) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    DpShared &S = *reinterpret_cast<DpShared *>(smem_raw);
    ColMeta *meta = reinterpret_cast<ColMeta *>(meta_all);
    uint16_t *seg = seg_all + (int64_t)blockIdx.x * C3B_PHASE_SEGMENT * seg_stride;
    const int tid = threadIdx.x;
    for (int64_t bi = blockIdx.x; bi < B.n_blocks; bi += gridDim.x) {
        const int64_t b = B.order[bi];
        const int64_t c0 = B.col_off[b], m = B.col_off[b + 1] - c0, r0 = B.read_off[b], nr = B.read_off[b + 1] - r0;
        const int64_t slot = 1ll << (B.kmax[b] - 1);
        uint32_t *ck = ckpt + B.ckpt_off[b];
        const int64_t n_seg = (m + C3B_PHASE_SEGMENT - 1) / C3B_PHASE_SEGMENT;
        if (tid == 0) { S.kprev = 0; S.nxt = 0; S.bad = 0; }
        __syncthreads();
        // ---- forward: the shapes of the columns, D, and the checkpoints
        for (int64_t j = 0; j < m; ++j) {
            if (tid == 0) {
                int na = 0, ns = 0;
                int32_t nact[C3B_PHASE_MAX_READS + 1];
                uint32_t sh = 0, lv = 0;
                for (int i = 0; i < S.kprev; ++i) {
                    if (B.read_last[r0 + S.act[i]] >= j) { sh |= 1u << i; nact[na++] = S.act[i]; }
                    else lv |= 1u << i;
                }
                ns = na;
                while (S.nxt < nr && B.read_first[r0 + S.nxt] == j) {
                    if (na == C3B_PHASE_MAX_READS) { S.bad = 1; break; }
                    nact[na++] = S.nxt++;
                }
                if (na == 0 || (j > 0 && ns == 0)) S.bad = 1;       // a block's columns are linked: some read spans each step
                for (int i = 0; i < na; ++i) S.act[i] = nact[i];
                S.meta = ColMeta{(uint16_t)na, (uint16_t)ns, (uint16_t)sh, (uint16_t)lv};
                meta[c0 + j] = S.meta;
                const int64_t e0 = B.ent_off[c0 + j];
                S.ne = (int)(B.ent_off[c0 + j + 1] - e0);
                if (S.ne > na) S.bad = 1;
                for (int e = 0; e < S.ne && !S.bad; ++e) {
                    int at = -1;
                    for (int i = 0; i < na; ++i) if (S.act[i] == B.ent_read[e0 + e]) at = i;
                    if (at < 0) { S.bad = 1; break; }
                    S.eb[e] = ebit[e0 + e] = (uint8_t)at;
                    S.ea[e] = B.ent_allele[e0 + e];
                    S.ew[e] = B.ent_weight[e0 + e];
                }
                if (S.meta.k > B.kmax[b]) S.bad = 1;
            }
            __syncthreads();
            if (S.bad) break;
            dp_column(S, j == 0, nullptr);
            if ((j + 1) % C3B_PHASE_SEGMENT == 0 && j + 1 < m)
                for (int s = tid; s < (1 << (S.meta.k - 1)); s += kThreads) ck[(j / C3B_PHASE_SEGMENT) * slot + s] = S.D[s];
            if (tid == 0) S.kprev = S.meta.k;
            __syncthreads();
        }
        if (S.bad) {
            if (tid == 0) atomicCAS(reinterpret_cast<unsigned long long *>(status), 0ull, (unsigned long long)(b + 1));
            __syncthreads();
            continue;
        }
        // ---- the optimum at the last column: the lowest state of the lowest D
        unsigned long long best = ~0ull;
        for (int s = tid; s < (1 << (S.meta.k - 1)); s += kThreads) {
            const unsigned long long x = (unsigned long long)S.D[s] << 32 | (unsigned)s;
            best = x < best ? x : best;
        }
        for (int d = 16; d; d >>= 1) {
            const unsigned long long o = __shfl_down_sync(0xffffffffu, best, d);
            best = o < best ? o : best;
        }
        if ((tid & 31) == 0) S.red[tid >> 5] = best;
        __syncthreads();
        if (tid < 32) {
            best = S.red[tid];
            for (int d = 16; d; d >>= 1) {
                const unsigned long long o = __shfl_down_sync(0xffffffffu, best, d);
                best = o < best ? o : best;
            }
        }
        // thread 0 keeps the backtrace's state (normalized index and whether its parts are swapped against the last column's)
        uint32_t st = (uint32_t)best, flip = 0;
        if (tid == 0) cost[b] = (int64_t)(best >> 32);
        __syncthreads();
        // ---- backtrace, segment by segment from the last
        for (int64_t g = n_seg - 1; g >= 0; --g) {
            const int64_t j0 = g * C3B_PHASE_SEGMENT, j1 = j0 + C3B_PHASE_SEGMENT < m ? j0 + C3B_PHASE_SEGMENT : m;
            if (g > 0) {
                const int kp = meta[c0 + j0 - 1].k;
                for (int s = tid; s < (1 << (kp - 1)); s += kThreads) S.D[s] = ck[(g - 1) * slot + s];
                if (tid == 0) S.kprev = kp;
            }
            for (int64_t j = j0; j < j1; ++j) {
                if (tid == 0) {
                    S.meta = meta[c0 + j];
                    load_entries(S, B, ebit, c0 + j);
                }
                __syncthreads();
                dp_column(S, j == 0, seg + (j - j0) * seg_stride);
                if (tid == 0) S.kprev = S.meta.k;
                __syncthreads();
            }
            if (tid == 0) {
                for (int64_t j = j1 - 1; j >= j0; --j) {
                    S.meta = meta[c0 + j];
                    load_entries(S, B, ebit, c0 + j);
                    uint32_t total = 0;
                    for (int e = 0; e < S.ne; ++e) total += S.ew[e];
                    const uint32_t o1 = opt1_of(S, st << 1);
                    hap[c0 + j] = (uint8_t)((o1 > total - o1) ^ flip);
                    if (j == 0) break;
                    const ColMeta cm = S.meta;
                    const uint32_t t = st & ((1u << (cm.ns - 1)) - 1);
                    const uint32_t l = seg[(j - j0) * seg_stride + t];
                    uint32_t full = deposit(t << 1, cm.sh) | deposit(l, cm.lv);
                    if (full & 1) {
                        full = ~full & ((1u << meta[c0 + j - 1].k) - 1);
                        flip ^= 1;
                    }
                    st = full >> 1;
                }
            }
            __syncthreads();
        }
        // ---- haplotype 0 carries allele 0 at the block's first column
        const uint8_t h0 = hap[c0];
        __syncthreads();
        for (int64_t j = tid; j < m; j += kThreads) hap[c0 + j] ^= h0;
        __syncthreads();
    }
}

}  // namespace

extern "C" int c3b_phase_dp_attributes(int *registers, int64_t *shared_bytes, int64_t *local_bytes, int *max_threads) {
    cudaFuncAttributes a;
    C3B_CUDA(cudaFuncGetAttributes(&a, phase_dp_kernel));
    if (registers) *registers = a.numRegs;
    if (shared_bytes) *shared_bytes = (int64_t)sizeof(DpShared);
    if (local_bytes) *local_bytes = (int64_t)a.localSizeBytes;
    if (max_threads) *max_threads = a.maxThreadsPerBlock;
    return 0;
}

static int frag_args(const char *who, const c3b_fa_records *rec, int64_t lo, int64_t hi, const c3b_phase_variants *v,
                     FragArgs &a) {
    if (!rec || !v || (v->n > 0 && (!v->pos || !v->ref || !v->alt)) || v->n < 0) {
        c3b_set_error("%s: null argument", who);
        return 1;
    }
    const c3b_bam_records &c = rec->core;
    if (c.n_reads > 0 && (!c.pos || !c.flag || !c.mapq || !c.cigar_off || !c.cigar || !c.seq_off || !c.seq || !c.l_qseq ||
                          !rec->qual || !rec->qual_off)) {
        c3b_set_error("%s: null record array (the records need their qualities: decode with fa_fields)", who);
        return 1;
    }
    a.r = C3bReads{c.n_reads, c.pos, c.flag, c.mapq, c.cigar_off, c.cigar, c.seq_off, c.seq, c.l_qseq, rec->qual_off, rec->qual,
                   nullptr, nullptr, nullptr, nullptr};
    a.lo = lo;
    a.hi = hi;
    a.v = *v;
    a.first = a.read_base = 0;
    return 0;
}

extern "C" int c3b_phase_count(const c3b_fa_records *records, int64_t lo, int64_t hi, const c3b_phase_variants *variants,
                               int64_t *offsets, int64_t *n_entries, int64_t *first, void *cuda_stream) {
    FragArgs a;
    if (frag_args("c3b_phase_count", records, lo, hi, variants, a)) return 1;
    if (!offsets || !n_entries || !first) {
        c3b_set_error("c3b_phase_count: null offsets / n_entries / first");
        return 1;
    }
    cudaStream_t s = (cudaStream_t)cuda_stream;
    const int64_t n = a.r.n;
    // the records' check, as every consumer of device records makes it
    uint64_t fault = C3B_REC_OK;
    {
        C3bBuf key(C3bBuf::exact);
        if (c3b_records_check_device(c3b_records_view(&records->core, records), key, s, &fault)) return 1;
        if (fault == C3B_REC_OK) fault = c3b_records_pairs(records);
    }
    if (fault != C3B_REC_OK) {
        c3b_set_error("c3b_phase_count: records: read %lld: %s", (long long)c3b_records_fault_read(fault), c3b_records_fault_text(fault));
        return 1;
    }
    int64_t host[2] = {0, 0};
    if (n == 0 || a.v.n == 0) {
        C3B_CUDA(cudaMemsetAsync(offsets, 0, (size_t)(n + 1) * 8, s));
        C3B_CUDA(cudaStreamSynchronize(s));
        *n_entries = 0;
        *first = 0;
        return 0;
    }
    // the counts go to offsets[1 .. n] and the first record's index to offsets[0], which is read back before the scan turns
    // offsets[1 ..] in place into the exclusive sums at offsets[0 .. n) and the total at offsets[n]
    const unsigned blocks = (unsigned)((n * 32 + 255) / 256);
    phase_fragment_kernel<false><<<blocks, 256, 0, s>>>(a, offsets + 1, nullptr, nullptr, nullptr, nullptr, nullptr, offsets);
    C3B_CUDA(cudaGetLastError());
    C3B_CUDA(cudaMemcpyAsync(&host[1], offsets, 8, cudaMemcpyDeviceToHost, s));
    block_scan_sum(offsets + 1, offsets, n, nullptr, offsets + n, s);
    C3B_CUDA(cudaGetLastError());
    C3B_CUDA(cudaMemcpyAsync(&host[0], offsets + n, 8, cudaMemcpyDeviceToHost, s));
    C3B_CUDA(cudaStreamSynchronize(s));
    *n_entries = host[0];
    *first = host[1];
    return 0;
}

extern "C" int c3b_phase_write(const c3b_fa_records *records, int64_t lo, int64_t hi, const c3b_phase_variants *variants,
                               const int64_t *offsets, int64_t first, int64_t read_base, int64_t *out_read, int32_t *out_var,
                               uint8_t *out_allele, uint8_t *out_weight, void *cuda_stream) {
    FragArgs a;
    if (frag_args("c3b_phase_write", records, lo, hi, variants, a)) return 1;
    if (a.r.n == 0 || a.v.n == 0) return 0;
    if (!offsets || !out_read || !out_var || !out_allele || !out_weight) {
        c3b_set_error("c3b_phase_write: null output");
        return 1;
    }
    a.first = first;
    a.read_base = read_base;
    const unsigned blocks = (unsigned)((a.r.n * 32 + 255) / 256);
    phase_fragment_kernel<true><<<blocks, 256, 0, (cudaStream_t)cuda_stream>>>(a, nullptr, offsets, out_read, out_var, out_allele,
                                                                               out_weight, nullptr);
    C3B_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int c3b_phase_dp(const c3b_phase_blocks *blocks, int n_ctas, uint8_t *hap, int64_t *cost, uint32_t *ckpt, uint16_t *seg,
                            int64_t seg_stride, uint16_t *meta, uint8_t *ebit, int64_t *status, void *cuda_stream) {
    if (!blocks || blocks->n_blocks < 0 || !status) {
        c3b_set_error("c3b_phase_dp: null argument");
        return 1;
    }
    cudaStream_t s = (cudaStream_t)cuda_stream;
    C3B_CUDA(cudaMemsetAsync(status, 0, 8, s));
    if (blocks->n_blocks == 0) return 0;
    if (n_ctas < 1 || !hap || !cost || !ckpt || !seg || !meta || !ebit || seg_stride < 1) {
        c3b_set_error("c3b_phase_dp: null output or no CTA");
        return 1;
    }
    const int grid = (int64_t)n_ctas < blocks->n_blocks ? n_ctas : (int)blocks->n_blocks;
    const size_t smem = sizeof(DpShared);
    C3B_CUDA(cudaFuncSetAttribute(phase_dp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    phase_dp_kernel<<<grid, kThreads, smem, s>>>(*blocks, hap, cost, ckpt, seg, seg_stride, meta, ebit, status);
    C3B_CUDA(cudaGetLastError());
    return 0;
}
