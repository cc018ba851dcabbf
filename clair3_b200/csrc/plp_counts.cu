// plp_counts.cu - the pileup feature counter on the GPU (include/clair3_b200_pileup.h; SURVEY.md 8f row N4, pileup half).
//
// Reference: calculate_clair3_pileup(), HKU-BAL/Clair3 src/clair3_pileup.c:142-476 - a column-by-column loop over htslib's
// bam_mplp_auto() with one incremental CIGAR cursor per read.  Here the work is turned around for a machine with 132 SMs and no
// cheap serial cursor:
//
//   K1 plp_scan_reads    one warp per read: read filter (src/medaka_bamiter.c:21-24) and a warp prefix sum over its CIGAR words ->
//                        per operation the reference offset of its END and the query offset of its START (int32, 8 B per word).
//                        With these every (read, position) pair can be resolved on its own, in any order: the operation on
//                        position p is the first one whose end offset exceeds p - pos (binary search), and htslib's
//                        resolve_cigar2 (is_del / is_refskip / indel / qpos) is a pure function of that operation and its
//                        neighbours.
//   K2 plp_prefix_max    running maximum of the read ends (reads are sorted by start, not by end): the reads that can touch a
//                        column tile are [first i with pmax[i] > tile start, first i with pos[i] >= tile end).
//   K3 plp_count_tile    one CTA per tile of 256 columns, ONE THREAD PER COLUMN.  The thread walks the tile's reads and owns every
//                        counter of its column - the 18 features (in shared memory, [feature][column], conflict-free), the
//                        deletion-length table and the insertion-string counters (a linked list of nodes in a shared-memory pool,
//                        spilling to a global pool) - so nothing on the counting path needs an atomic except pool allocation, and
//                        the per-column semantics are literally the reference's (strings compared base by base, no hashing).  The
//                        column's statistics and the allele-frequency test (float32 divisions as in the reference) follow.
//   K4 / K7 plp_scan_tiles   exclusive scan of the per-tile covered-column / candidate counts (htslib reports only covered columns,
//                        so the matrix is a compaction of the region).
//   K5 plp_emit          compaction: int64 rows (plp_data.matrix is size_t), major, stats, the 16-column flanking test.
//   K6 plp_quirk         the reference's index -1 quirk: a non-ACGT read base increments feature 17 of the PREVIOUS emitted column.
//   K8 plp_cands         candidate list, window starts and run bounds for c3b_forward_windows_bounded, and the reference's verdict
//                        on each candidate's window (plain, or with call_ht the zero-padded head / tail windows).
//
// Bound: HBM / L2 latency (integer work, no tensor cores).  Algorithmic bytes per call: 8 B per CIGAR word (read + offsets
// written and re-read), 0.5 B per aligned base (packed sequence), ~27 B per read, and per column 72 + 24 + 4 B dense (written, read
// once) + 144 + 8 + 24 B emitted: see DESIGN.md 3.8.
#include <limits.h>
#include <stdlib.h>
#include <string.h>

#include "c3b_internal.h"
#include "../../include/clair3_b200_pileup.h"

namespace {

constexpr int TILE = 256;
constexpr int NFEAT = 18;
constexpr int NCNT = 19;          // 18 features + the index -1 counter
constexpr int NP = 704;           // shared-memory indel nodes per tile (20 B each): 33.5 KB per CTA with the counters -> 6 CTAs per SM
constexpr int FLANK = 16;         // pileup_flanking_base_num, src/clair3_pileup.h:93
constexpr int G_POOL = 1 << 21;   // global overflow nodes per workspace
constexpr int AL_CAP = 1 << 22;   // exported allele records per call (16 B each)

struct DevReads {
    int64_t n;
    const int64_t *pos;
    const uint16_t *flag;
    const uint8_t *mapq;
    const int64_t *cigar_off;
    const uint32_t *cigar;
    const int64_t *seq_off;
    const uint8_t *seq;
    const int32_t *l_qseq;
};

__device__ __forceinline__ bool ref_cons(uint32_t op) { return (0x18Du >> op) & 1u; }   // M D N = X
__device__ __forceinline__ bool qry_cons(uint32_t op) { return (0x193u >> op) & 1u; }   // M I S = X
__device__ __forceinline__ int nib_at(const uint8_t *sq, int lq, long long i) {
    if (i < 0 || i >= lq) return 0;
    return (__ldg(sq + (i >> 1)) >> ((~i & 1) << 2)) & 15;
}

// ---------------------------------------------------------------------------------------------------------------- K1
__global__ void plp_scan_reads_kernel(DevReads R, int min_mq, int32_t *__restrict__ opx_end, int32_t *__restrict__ opy,
                                      int64_t *__restrict__ rend, int *status) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < R.n; r += nwarps) {
        const int64_t cb = R.cigar_off[r], ce = R.cigar_off[r + 1];
        long long cr = 0, cq = 0;
        for (int64_t base = cb; base < ce; base += 32) {
            const int64_t k = base + lane;
            const uint32_t c = k < ce ? R.cigar[k] : 0u;
            const uint32_t op = c & 15u;
            const long long l = (long long)(c >> 4);
            const long long rl = (k < ce && ref_cons(op)) ? l : 0, ql = (k < ce && qry_cons(op)) ? l : 0;
            long long ir = rl, iq = ql;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const long long a = __shfl_up_sync(0xffffffffu, ir, d), b = __shfl_up_sync(0xffffffffu, iq, d);
                if (lane >= d) { ir += a; iq += b; }
            }
            if (k < ce) {
                long long xe = cr + ir, y0 = cq + iq - ql;
                if (xe > INT_MAX || y0 > INT_MAX) {
                    atomicOr(status, 2);
                    xe = xe > INT_MAX ? INT_MAX : xe;
                    y0 = y0 > INT_MAX ? INT_MAX : y0;
                }
                opx_end[k] = (int32_t)xe;
                opy[k] = (int32_t)y0;
            }
            cr += __shfl_sync(0xffffffffu, ir, 31);
            cq += __shfl_sync(0xffffffffu, iq, 31);
        }
        if (lane == 0) {
            const bool keep = !(R.flag[r] & (4 | 256 | 512 | 1024 | 2048)) && (int)R.mapq[r] >= min_mq && cr > 0;
            rend[r] = R.pos[r] + (keep ? cr : 0);        // a dropped read covers nothing
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------- K2
__global__ void plp_prefix_max_kernel(const int64_t *__restrict__ rend, int64_t *__restrict__ pmax, int64_t n) {
    __shared__ long long wmax[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    long long carry = LLONG_MIN;
    for (int64_t base = 0; base < n; base += 1024) {
        const int64_t i = base + threadIdx.x;
        long long v = i < n ? (long long)rend[i] : LLONG_MIN;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const long long a = __shfl_up_sync(0xffffffffu, v, d);
            if (lane >= d && a > v) v = a;
        }
        if (lane == 31) wmax[warp] = v;
        __syncthreads();
        if (warp == 0) {
            long long t = wmax[lane];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const long long a = __shfl_up_sync(0xffffffffu, t, d);
                if (lane >= d && a > t) t = a;
            }
            wmax[lane] = t;
        }
        __syncthreads();
        if (warp > 0 && wmax[warp - 1] > v) v = wmax[warp - 1];
        if (carry > v) v = carry;
        if (i < n) pmax[i] = v;
        if (wmax[31] > carry) carry = wmax[31];
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------------------------------------------- K3
struct CountArgs {
    DevReads R;
    const int32_t *opx_end;
    const int32_t *opy;
    const int64_t *rend;
    const int64_t *pmax;
    int64_t start, end;
    const char *ref;
    int64_t ref_start, ref_len;
    c3b_plp_params prm;
    int32_t *rows32;      // [W][18] dense
    int32_t *dstats;      // [W][6]  depth, ref, alt, del, ins, flags (bit 0 pass_af before the flanking test, bit 2 covered)
    int32_t *nquirk;      // [W]
    int64_t *gv_ref;      // [W] or null
    int64_t *gv_tot;
    int32_t *tile_cov;    // [tiles]
    uint32_t *g_meta, *g_read, *g_qpos, *g_cnt;
    int32_t *g_next;
    int *g_used;
    int *status;
    // optional export of the candidate columns' allele lists (for the all_alt_info text): null = off
    uint32_t *al_meta, *al_read, *al_qpos, *al_cnt;
    int32_t *al_off, *al_n;   // [W] first record / number of records of a column
    int32_t *ins_last;        // [W] last read with an insertion on a candidate column, -1 = none
    int *al_used;
    int al_cap;
};

struct Pool {          // the tile's shared-memory indel nodes
    uint32_t *meta;    // bit 31 insertion, bit 30 reverse strand, length
    uint32_t *read;    // representative read
    uint32_t *qpos;    // first inserted base in that read
    uint32_t *cnt;
    int32_t *next;
    int *used;
};

#define NODE(arr, i) (*((i) < NP ? &P.arr[(i)] : &A.g_##arr[(i) - NP]))

// One indel allele seen on this thread's column (src/clair3_pileup.c:253-272 deletion table, :293-307 insertion strings): find it
// in the column's list (strings compared base by base against the representative read) or append it; update all / best.
// meta = insertion << 31 | reverse << 30 | length, q0 = first inserted base in read r (insertions).
__device__ __forceinline__ void plp_event(const CountArgs &A, const Pool &P, int32_t *cnt, const int tid, const uint32_t meta,
                                          const long long q0, const uint32_t r, int &head) {
    const int kind = (int)(meta >> 31), rev = (int)((meta >> 30) & 1u);
    const long long len = (long long)(meta & 0x3fffffffu);
    const uint8_t *sq = A.R.seq;
    int lq = 0;
    if (kind) {
        sq = A.R.seq + __ldg(A.R.seq_off + r);
        lq = __ldg(A.R.l_qseq + r);
    }
    int c = 0;
    bool found = false;
    for (int i = head; i >= 0; i = NODE(next, i)) {
        if (NODE(meta, i) != meta) continue;
        bool same = true;
        if (kind) {
            const uint32_t rr = NODE(read, i);
            const long long rq = (long long)NODE(qpos, i);
            const uint8_t *s2 = A.R.seq + __ldg(A.R.seq_off + rr);
            const int lq2 = __ldg(A.R.l_qseq + rr);
            for (long long j = 0; j < len; ++j)
                if (nib_at(sq, lq, q0 + j) != nib_at(s2, lq2, rq + j)) { same = false; break; }
        }
        if (same) { c = (int)(NODE(cnt, i) += 1u); found = true; break; }
    }
    if (!found) {
        int slot = atomicAdd(P.used, 1);
        if (slot >= NP) {
            const int g = atomicAdd(A.g_used, 1);
            if (g >= G_POOL) { atomicOr(A.status, 1); slot = -1; } else slot = NP + g;
        }
        if (slot >= 0) {
            NODE(meta, slot) = meta;
            NODE(read, slot) = r;
            NODE(qpos, slot) = (uint32_t)q0;
            NODE(cnt, slot) = 1u;
            NODE(next, slot) = head;
            head = slot;
        }
        c = 1;
    }
    const int f_all = kind ? (rev ? 13 : 4) : (rev ? 15 : 6);
    cnt[f_all * TILE + tid] += 1;                                            // stats.sum / all_count
    if (c > cnt[(f_all + 1) * TILE + tid]) cnt[(f_all + 1) * TILE + tid] = c;       // stats.max / best_count
}

// What ONE read shows on ONE column (htslib's resolve_cigar2 as a pure function of the operation k that covers the column) and
// what the reference's inner loop does with it (src/clair3_pileup.c:249-308).  cw / xend / y0 are operation k's CIGAR word, end
// offset and query start; nb is the read base at qpos.  Returns the indel allele that starts after this base, if any, in
// (ev_meta, ev_q0) instead of recording it (the caller records it).
__device__ __forceinline__ bool plp_visit(const CountArgs &A, int32_t *cnt, const int tid, const int64_t cb, const int nc,
                                          const int off, const int k, const uint32_t cw, const int xend, const int y0, const int rev,
                                          const int nb, int &depth, uint32_t &ev_meta, long long &ev_q0) {
    const uint32_t op = cw & 15u;
    const int l = (int)(cw >> 4);
    if (op == 3u) return false;                                              // is_refskip, src/clair3_pileup.c:251
    long long indel = 0;
    if (off == xend - 1 && k + 1 < nc) {                                     // resolve_cigar2: peek the next operation
        uint32_t c2 = __ldg(A.R.cigar + cb + k + 1);
        const uint32_t op2 = c2 & 15u;
        if (op2 == 2u && op != 2u) {
            indel = -(long long)(c2 >> 4);
            for (int j = k + 2; j < nc; ++j) {
                c2 = __ldg(A.R.cigar + cb + j);
                if ((c2 & 15u) == 2u) indel -= (long long)(c2 >> 4); else break;
            }
        } else if (op2 == 1u) {
            indel = (long long)(c2 >> 4);
            for (int j = k + 2; j < nc; ++j) {
                c2 = __ldg(A.R.cigar + cb + j);
                const uint32_t o = c2 & 15u;
                if (o == 1u) indel += (long long)(c2 >> 4); else if (o != 6u) break;
            }
        } else if (op2 == 6u && k + 2 < nc) {
            long long l3 = 0;
            for (int j = k + 2; j < nc; ++j) {
                c2 = __ldg(A.R.cigar + cb + j);
                const uint32_t o = c2 & 15u;
                if (o == 1u) l3 += (long long)(c2 >> 4); else if (ref_cons(o)) break;
            }
            if (l3 > 0) indel = l3;
        }
    }
    const bool is_del = (op == 2u);
    const long long qpos = is_del ? (long long)y0 : (long long)y0 + (off - (xend - l));

    // the column's base / deletion counters, src/clair3_pileup.c:276-290
    int base_i;
    if (is_del) {
        base_i = rev ? 17 : 8;
    } else {
        const int t = nb == 1 ? 0 : nb == 2 ? 1 : nb == 4 ? 2 : nb == 8 ? 3 : -1;
        base_i = t < 0 ? -1 : t + 9 * rev;
    }
    ++depth;
    cnt[(base_i >= 0 ? base_i : NFEAT) * TILE + tid] += 1;
    if (indel == 0) return false;
    const int kind = indel > 0 ? 1 : 0;
    long long len = indel > 0 ? indel : -indel;
    if (len >= (1ll << 30)) { atomicOr(A.status, 4); len = (1ll << 30) - 1; }
    ev_meta = ((uint32_t)kind << 31) | ((uint32_t)rev << 30) | (uint32_t)len;
    ev_q0 = qpos + (is_del ? 0 : 1);
    return true;
}

// Per-warp read ranges and six CTAs per SM keep enough reads in flight to hide the per-read CIGAR searches.
__global__ void __launch_bounds__(TILE, 6) plp_count_tile_kernel(CountArgs A) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    int32_t *cnt = reinterpret_cast<int32_t *>(smem_raw);                       // [NCNT][TILE]
    __shared__ int s_used;
    Pool P;
    P.meta = reinterpret_cast<uint32_t *>(cnt + NCNT * TILE);
    P.read = P.meta + NP;
    P.qpos = P.read + NP;
    P.cnt = P.qpos + NP;
    P.next = reinterpret_cast<int32_t *>(P.cnt + NP);
    P.used = &s_used;
    const int tid = threadIdx.x;
    const int64_t tile_start = A.start + (int64_t)blockIdx.x * TILE;
    const int64_t tile_end = tile_start + TILE < A.end ? tile_start + TILE : A.end;
    const int64_t p = tile_start + tid;
    const bool active = p < A.end;
#pragma unroll
    for (int f = 0; f < NCNT; ++f) cnt[f * TILE + tid] = 0;
    if (tid == 0) s_used = 0;
    __syncthreads();

    // reads that can touch this WARP's 32 columns (per tile the loop ran 1.7x as many warp iterations: a 256-column tile sees
    // reads that end before or start after most of its warps)
    int64_t lo, hi;
    {
        const int64_t w_start = tile_start + (tid & ~31);
        const int64_t w_end = w_start + 32 < tile_end ? w_start + 32 : tile_end;
        int64_t a = 0, b = w_start < tile_end ? A.R.n : 0;
        while (a < b) { const int64_t m = (a + b) >> 1; if (__ldg(A.pmax + m) > w_start) b = m; else a = m + 1; }
        lo = a;
        b = w_start < tile_end ? A.R.n : 0;
        while (a < b) { const int64_t m = (a + b) >> 1; if (__ldg(A.R.pos + m) >= w_end) b = m; else a = m + 1; }
        hi = a;
    }

    int depth = 0, head = -1;
    int ins_last = -1;       // the last read with an insertion here: did a put of a present key follow the last new string?
    bool covered = false;
    for (int64_t r = lo; r < hi; ++r) {                      // warp-uniform trip count
        const int64_t rp = __ldg(A.R.pos + r), re = __ldg(A.rend + r);
        const bool in = active && p >= rp && p < re;
        uint32_t e_meta = 0;
        long long e_q0 = 0;
        if (in) {
            covered = true;                                  // n_plp > 0: htslib reports the column
            const int64_t cb = __ldg(A.R.cigar_off + r);
            const int nc = (int)(__ldg(A.R.cigar_off + r + 1) - cb);
            const int off = (int)(p - rp);
            const int32_t *ox = A.opx_end + cb;
            int a = 0, b = nc;                               // the operation on this column: first one whose end offset exceeds off
            while (a < b) { const int m = (a + b) >> 1; if (__ldg(ox + m) > off) b = m; else a = m + 1; }
            const int k = a;
            const uint32_t cw = __ldg(A.R.cigar + cb + k);
            const int xend = __ldg(ox + k);
            const int y0 = __ldg(A.opy + cb + k);
            const int rev = (__ldg(A.R.flag + r) >> 4) & 1;
            const uint32_t op = cw & 15u;
            int nb = 0;
            if (op != 2u && op != 3u)
                nb = nib_at(A.R.seq + __ldg(A.R.seq_off + r), __ldg(A.R.l_qseq + r), (long long)y0 + (off - (xend - (int)(cw >> 4))));
            if (plp_visit(A, cnt, tid, cb, nc, off, k, cw, xend, y0, rev, nb, depth, e_meta, e_q0)) {
                plp_event(A, P, cnt, tid, e_meta, e_q0, (uint32_t)r, head);
                if (e_meta >> 31) ins_last = (int)r;
            }
        }
    }

    // the column's statistics and allele-frequency test, src/clair3_pileup.c:349-387
    if (active) {
        int32_t *ds = A.dstats + (p - A.start) * 6;
        if (covered) {
            const int del_count = cnt[6 * TILE + tid] + cnt[15 * TILE + tid];
            const int ins_count = cnt[4 * TILE + tid] + cnt[13 * TILE + tid];
            const int64_t ro = p - A.ref_start;
            int rb = (ro >= 0 && ro < A.ref_len) ? (int)(unsigned char)A.ref[ro] : 'N';
            if (rb >= 'a' && rb <= 'z') rb -= 32;
            const int bi = rb - 'A';
            const int rf = bi == 2 ? 1 : bi == 6 ? 2 : bi == 19 ? 3 : 0;          // base2index, src/clair3_pileup.h:57-62
            int fsum = 0, rsum = 0, ref_count = 0, alt_count = 0, all_alt = 0, major_alt = 0;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int cf = cnt[i * TILE + tid], cr = cnt[(i + 9) * TILE + tid];
                fsum += cf;
                rsum += cr;
                if (i == rf) {
                    ref_count = cf + cr;
                } else if (cf + cr > alt_count) {
                    alt_count = cf + cr;
                    major_alt = i == 0 ? 'A' : i == 1 ? 'C' : i == 2 ? 'G' : 'T';
                    all_alt += alt_count;
                }
            }
            cnt[rf * TILE + tid] = -fsum;
            cnt[(rf + 9) * TILE + tid] = -rsum;
            const int d = depth < 1 ? 1 : depth;
            const float fd = (float)d;
            const bool ref_acgt = rb == 'A' || rb == 'C' || rb == 'G' || rb == 'T';
            const bool snp = __fdiv_rn((float)alt_count, fd) >= A.prm.min_snp_af;
            bool pass;
            if (A.prm.call_snp_only) {
                pass = snp;
            } else {
                pass = ref_count < alt_count || ref_count < ins_count || ref_count < del_count ||
                       (ref_count > 0 && ref_count == alt_count && rb - major_alt < 0) || snp;
                pass = pass || __fdiv_rn((float)del_count, fd) >= A.prm.min_indel_af ||
                       __fdiv_rn((float)ins_count, fd) >= A.prm.min_indel_af;
            }
            pass = pass && (int64_t)d >= A.prm.min_depth && ref_acgt;
            ds[0] = d; ds[1] = ref_count; ds[2] = alt_count; ds[3] = del_count; ds[4] = ins_count;
            ds[5] = (pass ? 1 : 0) | 4;
            if (A.al_meta) {               // the column's distinct alleles, oldest first (the list is newest first)
                int n = 0;
                if (pass)
                    for (int i = head; i >= 0; i = NODE(next, i)) ++n;
                int base = n ? atomicAdd(A.al_used, n) : 0;
                if (base + n > A.al_cap) { atomicOr(A.status, 8); n = 0; base = 0; }
                A.al_off[p - A.start] = base;
                A.al_n[p - A.start] = n;
                A.ins_last[p - A.start] = pass ? ins_last : -1;
                int wr = base + n - 1;
                for (int i = head; i >= 0 && wr >= base; i = NODE(next, i), --wr) {
                    A.al_meta[wr] = NODE(meta, i);
                    A.al_read[wr] = NODE(read, i);
                    A.al_qpos[wr] = NODE(qpos, i);
                    A.al_cnt[wr] = NODE(cnt, i);
                }
            }
            if (A.gv_ref) {
                A.gv_ref[p - A.start] = ref_count;
                A.gv_tot[p - A.start] = (int64_t)ref_count + all_alt + del_count + ins_count;
            }
        } else {
            ds[0] = ds[1] = ds[2] = ds[3] = ds[4] = ds[5] = 0;
            if (A.al_meta) { A.al_off[p - A.start] = 0; A.al_n[p - A.start] = 0; A.ins_last[p - A.start] = -1; }
        }
        A.nquirk[p - A.start] = cnt[NFEAT * TILE + tid];
    }
    const int ncov = __syncthreads_count(active && covered);
    if (tid == 0) A.tile_cov[blockIdx.x] = ncov;
    // dense rows, coalesced: the tile's [columns][18] block is contiguous
    const int ncol_t = (int)(tile_end - tile_start);
    int32_t *dst = A.rows32 + (tile_start - A.start) * NFEAT;
    for (int e = tid; e < ncol_t * NFEAT; e += TILE) {
        const int c = e / NFEAT, f = e - c * NFEAT;
        dst[e] = cnt[f * TILE + c];
    }
}

// ---------------------------------------------------------------------------------------------------------------- K4 / K7
__global__ void plp_scan_tiles_kernel(const int32_t *__restrict__ cnt, int64_t *__restrict__ off, int n, int64_t *total) {
    __shared__ long long wsum[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    long long carry = 0;
    for (int base = 0; base < n; base += 1024) {
        const int i = base + threadIdx.x;
        const long long own = i < n ? (long long)cnt[i] : 0;
        long long v = own;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const long long a = __shfl_up_sync(0xffffffffu, v, d);
            if (lane >= d) v += a;
        }
        if (lane == 31) wsum[warp] = v;
        __syncthreads();
        if (warp == 0) {
            long long t = wsum[lane];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const long long a = __shfl_up_sync(0xffffffffu, t, d);
                if (lane >= d) t += a;
            }
            wsum[lane] = t;
        }
        __syncthreads();
        const long long incl = v + (warp > 0 ? wsum[warp - 1] : 0) + carry;
        if (i < n) off[i] = incl - own;
        carry += wsum[31];
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = carry;
}

// ---------------------------------------------------------------------------------------------------------------- K5
struct EmitArgs {
    int64_t start, end;
    int call_ht;
    const int32_t *rows32;
    const int32_t *dstats;
    const int64_t *tile_off;
    int64_t *matrix;
    int64_t *major;
    int32_t *stats;
    int32_t *dci;         // [W] emitted column index of a position, -1 = not covered
    int32_t *tile_cand;
};

__global__ void __launch_bounds__(TILE) plp_emit_kernel(EmitArgs A) {
    __shared__ int32_t rows_s[TILE * NFEAT];
    __shared__ int map_s[TILE];
    __shared__ int wsum[TILE / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t tile_start = A.start + (int64_t)blockIdx.x * TILE;
    const int64_t tile_end = tile_start + TILE < A.end ? tile_start + TILE : A.end;
    const int64_t p = tile_start + tid;
    const bool active = p < A.end;
    const int ncol_t = (int)(tile_end - tile_start);
    const int32_t *src = A.rows32 + (tile_start - A.start) * NFEAT;
    for (int e = tid; e < ncol_t * NFEAT; e += TILE) rows_s[e] = src[e];
    const int flags = active ? A.dstats[(p - A.start) * 6 + 5] : 0;
    const bool covered = (flags & 4) != 0;
    const unsigned bal = __ballot_sync(0xffffffffu, covered);
    if (lane == 0) wsum[warp] = __popc(bal);
    __syncthreads();
    int pre = 0, ntile = 0;
#pragma unroll
    for (int w = 0; w < TILE / 32; ++w) {
        if (w < warp) pre += wsum[w];
        ntile += wsum[w];
    }
    const int lci = pre + __popc(bal & ((1u << lane) - 1u));
    const int64_t t_off = A.tile_off[blockIdx.x];
    bool cand = false;
    if (covered) {
        const int64_t ci = t_off + lci;
        map_s[lci] = tid;
        A.major[ci] = p;
        A.dci[p - A.start] = (int32_t)ci;
        cand = (flags & 1) != 0;
        if (cand && !A.call_ht) {        // contiguous_flanking_num >= 16 (src/clair3_pileup.c:227-231, 385-387), pre_pos == 0 quirk included
            const int64_t lo = p - FLANK;
            cand = lo >= (A.start > 1 ? A.start : 1);
            for (int64_t q = lo; cand && q < p; ++q) cand = (A.dstats[(q - A.start) * 6 + 5] & 4) != 0;
        }
        bool zero = true;
#pragma unroll
        for (int f = 0; f < NFEAT; ++f) zero = zero && rows_s[tid * NFEAT + f] == 0;
        const int32_t *ds = A.dstats + (p - A.start) * 6;
        int32_t *st = A.stats + ci * 6;
        st[0] = ds[0]; st[1] = ds[1]; st[2] = ds[2]; st[3] = ds[3]; st[4] = ds[4];
        st[5] = (cand ? 1 : 0) | (zero ? 2 : 0);
    } else if (active) {
        A.dci[p - A.start] = -1;
    }
    const int ncand = __syncthreads_count(cand);
    if (tid == 0) A.tile_cand[blockIdx.x] = ncand;
    int64_t *dst = A.matrix + t_off * NFEAT;
    for (int e = tid; e < ntile * NFEAT; e += TILE) {
        const int c = e / NFEAT, f = e - c * NFEAT;
        dst[e] = (int64_t)rows_s[map_s[c] * NFEAT + f];
    }
}

// ---------------------------------------------------------------------------------------------------------------- K6
__global__ void plp_quirk_kernel(const int64_t *n_cols_dev, const int64_t *__restrict__ major, const int32_t *__restrict__ nquirk,
                                 int64_t start, int64_t *matrix, int32_t *stats) {
    const int64_t ci = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t n = *n_cols_dev;
    if (ci + 1 < n) {
        const int q = nquirk[major[ci + 1] - start];
        if (q > 0) {                      // matrix[major_col - 1] += 1 per non-ACGT read base of the NEXT emitted column
            matrix[ci * NFEAT + 17] += q;
            stats[ci * 6 + 5] &= ~2;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------- K8
struct CandArgs {
    int64_t start, end;
    int call_ht;
    const int64_t *n_cols_dev;
    const int32_t *dci;
    const int32_t *stats;
    const int64_t *major;
    const int64_t *tile_coff;
    int64_t *cand_cols;
    int64_t *wstart;
    int64_t *wbounds;     // [n_cand][2]: the window rows [lo, hi) inside the candidate's contiguous run
    uint8_t *cand_ok;
};

__global__ void __launch_bounds__(TILE) plp_cands_kernel(CandArgs A) {
    __shared__ int wsum[TILE / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t p = A.start + (int64_t)blockIdx.x * TILE + tid;
    const int64_t n = *A.n_cols_dev;
    int64_t ci = -1;
    if (p < A.end) ci = A.dci[p - A.start];
    const bool cand = ci >= 0 && (A.stats[ci * 6 + 5] & 1);
    const unsigned bal = __ballot_sync(0xffffffffu, cand);
    if (lane == 0) wsum[warp] = __popc(bal);
    __syncthreads();
    int pre = 0;
#pragma unroll
    for (int w = 0; w < TILE / 32; ++w)
        if (w < warp) pre += wsum[w];
    if (cand) {
        const int64_t j = A.tile_coff[blockIdx.x] + pre + __popc(bal & ((1u << lane) - 1u));
        A.cand_cols[j] = ci;
        A.wstart[j] = ci - FLANK;
        // preprocess/CreateTensorPileupFromCffi.py:356-396 over the contiguous chunks of :180-236 (oracle/pileup_oracle.c states
        // it line by line): the candidate's run of consecutive positions, looked at from row ci - 16 to row ci + 18
        int64_t lo = ci, hi = ci;
        while (lo > ci - FLANK && lo > 0 && A.major[lo - 1] == A.major[lo] - 1) --lo;
        while (hi < ci + FLANK + 2 && hi + 1 < n && A.major[hi + 1] == A.major[hi] + 1) ++hi;
        const bool head_full = lo == ci - FLANK;
        bool ok;
        if (head_full && hi == ci + FLANK + 2) {            // :358 the run reaches two rows past the window; :365 no all-zero row
            ok = true;
            for (int64_t q = ci - FLANK; ok && q <= ci + FLANK; ++q) ok = (A.stats[q * 6 + 5] & 2) == 0;
        } else {                                            // :370-396 head / tail windows, zero-padded, no all-zero test
            ok = A.call_ht && hi > ci && (head_full || hi >= ci + FLANK);
        }
        A.cand_ok[j] = ok ? 1 : 0;
        A.wbounds[2 * j] = lo;
        A.wbounds[2 * j + 1] = (hi < ci + FLANK ? hi : ci + FLANK) + 1;
    }
}

struct DBuf : C3bBuf {
    int ensure(size_t bytes) { return C3bBuf::ensure(bytes, "c3b_plp"); }
};

}  // namespace

struct c3b_plp {
    int device = 0;
    // inputs (copies of host records)
    DBuf in_pos, in_flag, in_mapq, in_coff, in_cigar, in_soff, in_seq, in_lq, in_ref;
    // scratch
    DBuf opx, opy, rend, pmax, rows32, dstats, nquirk, dci, tile_cov, tile_off, tile_cand, tile_coff;
    DBuf g_meta, g_read, g_qpos, g_cnt, g_next;
    DBuf al_meta, al_read, al_qpos, al_cnt, al_off, al_n, ins_last;   // allele export (params.alt_info)
    DBuf counters;      // int64 n_cols, int64 n_cand, int g_used, int status
    // outputs
    DBuf matrix, major, stats, cand_cols, wstart, wbounds, cand_ok, gv_ref, gv_tot;
    int64_t W = 0;
    bool gvcf = false, counted = false, alleles = false;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    int launches = 0;
    int64_t *host_counters = nullptr;   // pinned: n_cols, n_cand, (g_used | status << 32)
    int64_t n_cols = -1, n_cand = -1;
};

extern "C" {

int c3b_plp_create(c3b_plp **out, int device_ordinal) {
    if (!out) { c3b_set_error("c3b_plp_create: null out"); return 1; }
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) {
        c3b_set_error("no CUDA device: %s (clair3_b200 has no CPU fallback)", cudaGetErrorString(e));
        return 1;
    }
    if (device_ordinal < 0 || device_ordinal >= ndev) { c3b_set_error("bad device ordinal %d", device_ordinal); return 1; }
    cudaDeviceProp prop;
    C3B_CUDA(cudaGetDeviceProperties(&prop, device_ordinal));
    if (prop.major != 9 || prop.minor != 0) {
        c3b_set_error("device %d is sm_%d%d; this library contains only sm_90a code", device_ordinal, prop.major, prop.minor);
        return 1;
    }
    C3B_CUDA(cudaSetDevice(device_ordinal));
    c3b_plp *w = new c3b_plp();
    w->device = device_ordinal;
    if (cudaEventCreate(&w->ev0) != cudaSuccess || cudaEventCreate(&w->ev1) != cudaSuccess ||
        cudaMallocHost((void **)&w->host_counters, 4 * sizeof(int64_t)) != cudaSuccess) {
        c3b_set_error("c3b_plp_create: event / pinned allocation failed");
        delete w;
        return 1;
    }
    *out = w;
    return 0;
}

static int plp_upload(DBuf &b, const void *src, size_t bytes, int on_device, const void **dev, cudaStream_t s) {
    return c3b_upload(b, src, bytes, on_device, dev, s, "c3b_plp");
}

int c3b_plp_count(c3b_plp *w, const c3b_bam_records *reads, int on_device, int64_t start, int64_t end, const char *ref_seq,
                  int64_t ref_start, int64_t ref_len, const c3b_plp_params *params, void *cuda_stream) {
    if (!w || !reads || !params) { c3b_set_error("c3b_plp_count: null argument"); return 1; }
    if (end < start) { c3b_set_error("c3b_plp_count: end < start"); return 1; }
    if (end - start > (int64_t)INT_MAX / 32) { c3b_set_error("c3b_plp_count: region of %lld columns is too large for one call", (long long)(end - start)); return 1; }
    const int64_t n = reads->n_reads;
    if (n < 0 || n >= (int64_t)UINT_MAX) { c3b_set_error("c3b_plp_count: bad n_reads"); return 1; }
    if (n > 0 && (!reads->pos || !reads->flag || !reads->mapq || !reads->cigar_off || !reads->cigar || !reads->seq_off || !reads->seq || !reads->l_qseq)) {
        c3b_set_error("c3b_plp_count: null record array");
        return 1;
    }
    if (ref_len > 0 && !ref_seq) { c3b_set_error("c3b_plp_count: null ref_seq"); return 1; }
    C3B_CUDA(cudaSetDevice(w->device));
    cudaStream_t s = (cudaStream_t)cuda_stream;
    w->stream = s;
    w->counted = false;
    w->n_cols = w->n_cand = -1;
    const int64_t W = end - start;
    w->W = W;
    w->gvcf = params->gvcf != 0;
    const int tiles = (int)((W + TILE - 1) / TILE);

    // inputs
    DevReads R;
    memset(&R, 0, sizeof(R));
    R.n = n;
    int64_t n_cigar = 0, n_seq = 0;
    if (n > 0) {
        if (on_device) {
            C3B_CUDA(cudaMemcpyAsync(&n_cigar, reads->cigar_off + n, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
            C3B_CUDA(cudaMemcpyAsync(&n_seq, reads->seq_off + n, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
            C3B_CUDA(cudaStreamSynchronize(s));
        } else {
            n_cigar = reads->cigar_off[n];
            n_seq = reads->seq_off[n];
        }
        if (n_cigar < 0 || n_seq < 0) { c3b_set_error("c3b_plp_count: negative offsets"); return 1; }
        const void *d;
        if (plp_upload(w->in_pos, reads->pos, n * 8, on_device, &d, s)) return 1; R.pos = (const int64_t *)d;
        if (plp_upload(w->in_flag, reads->flag, n * 2, on_device, &d, s)) return 1; R.flag = (const uint16_t *)d;
        if (plp_upload(w->in_mapq, reads->mapq, n, on_device, &d, s)) return 1; R.mapq = (const uint8_t *)d;
        if (plp_upload(w->in_coff, reads->cigar_off, (n + 1) * 8, on_device, &d, s)) return 1; R.cigar_off = (const int64_t *)d;
        if (plp_upload(w->in_cigar, reads->cigar, n_cigar * 4, on_device, &d, s)) return 1; R.cigar = (const uint32_t *)d;
        if (plp_upload(w->in_soff, reads->seq_off, (n + 1) * 8, on_device, &d, s)) return 1; R.seq_off = (const int64_t *)d;
        if (plp_upload(w->in_seq, reads->seq, n_seq, on_device, &d, s)) return 1; R.seq = (const uint8_t *)d;
        if (plp_upload(w->in_lq, reads->l_qseq, n * 4, on_device, &d, s)) return 1; R.l_qseq = (const int32_t *)d;
    }
    const void *dref = nullptr;
    if (plp_upload(w->in_ref, ref_seq, (size_t)(ref_len > 0 ? ref_len : 0), on_device, &dref, s)) return 1;

    // scratch and outputs
    const size_t Wz = (size_t)(W > 0 ? W : 1), Tz = (size_t)(tiles > 0 ? tiles : 1);
    if (w->opx.ensure((size_t)(n_cigar + 1) * 4) || w->opy.ensure((size_t)(n_cigar + 1) * 4) || w->rend.ensure((size_t)(n + 1) * 8) ||
        w->pmax.ensure((size_t)(n + 1) * 8) || w->rows32.ensure(Wz * NFEAT * 4) || w->dstats.ensure(Wz * 6 * 4) ||
        w->nquirk.ensure(Wz * 4) || w->dci.ensure(Wz * 4) || w->tile_cov.ensure(Tz * 4) || w->tile_off.ensure(Tz * 8) ||
        w->tile_cand.ensure(Tz * 4) || w->tile_coff.ensure(Tz * 8) || w->g_meta.ensure((size_t)G_POOL * 4) ||
        w->g_read.ensure((size_t)G_POOL * 4) || w->g_qpos.ensure((size_t)G_POOL * 4) || w->g_cnt.ensure((size_t)G_POOL * 4) ||
        w->g_next.ensure((size_t)G_POOL * 4) || w->counters.ensure(32) || w->matrix.ensure(Wz * NFEAT * 8) ||
        w->major.ensure(Wz * 8) || w->stats.ensure(Wz * 6 * 4) || w->cand_cols.ensure(Wz * 8) || w->wstart.ensure(Wz * 8) ||
        w->wbounds.ensure(Wz * 16) || w->cand_ok.ensure(Wz))
        return 1;
    if (w->gvcf && (w->gv_ref.ensure(Wz * 8) || w->gv_tot.ensure(Wz * 8))) return 1;
    w->alleles = params->alt_info != 0;
    if (w->alleles && (w->al_meta.ensure((size_t)AL_CAP * 4) || w->al_read.ensure((size_t)AL_CAP * 4) || w->al_qpos.ensure((size_t)AL_CAP * 4) ||
                       w->al_cnt.ensure((size_t)AL_CAP * 4) || w->al_off.ensure(Wz * 4) || w->al_n.ensure(Wz * 4) ||
                       w->ins_last.ensure(Wz * 4)))
        return 1;
    C3B_CUDA(cudaMemsetAsync(w->counters.p, 0, 32, s));
    if (w->gvcf && W > 0) {
        C3B_CUDA(cudaMemsetAsync(w->gv_ref.p, 0, (size_t)W * 8, s));
        C3B_CUDA(cudaMemsetAsync(w->gv_tot.p, 0, (size_t)W * 8, s));
    }
    int64_t *n_cols_dev = w->counters.as<int64_t>();
    int64_t *n_cand_dev = n_cols_dev + 1;
    int *g_used = reinterpret_cast<int *>(n_cols_dev + 2);
    int *status = g_used + 1;
    int *al_used = reinterpret_cast<int *>(n_cols_dev + 3);

    w->launches = 0;
    C3B_CUDA(cudaEventRecord(w->ev0, s));
    if (W > 0) {
        if (n > 0) {
            int blocks = (int)((n * 32 + 255) / 256);
            if (blocks > 132 * 8) blocks = 132 * 8;
            plp_scan_reads_kernel<<<blocks, 256, 0, s>>>(R, params->min_mq, w->opx.as<int32_t>(), w->opy.as<int32_t>(), w->rend.as<int64_t>(), status);
            plp_prefix_max_kernel<<<1, 1024, 0, s>>>(w->rend.as<int64_t>(), w->pmax.as<int64_t>(), n);
            w->launches += 2;
        }
        CountArgs A;
        A.R = R;
        A.opx_end = w->opx.as<int32_t>(); A.opy = w->opy.as<int32_t>(); A.rend = w->rend.as<int64_t>(); A.pmax = w->pmax.as<int64_t>();
        A.start = start; A.end = end; A.ref = (const char *)dref; A.ref_start = ref_start; A.ref_len = ref_len > 0 ? ref_len : 0;
        A.prm = *params;
        A.rows32 = w->rows32.as<int32_t>(); A.dstats = w->dstats.as<int32_t>(); A.nquirk = w->nquirk.as<int32_t>();
        A.gv_ref = w->gvcf ? w->gv_ref.as<int64_t>() : nullptr; A.gv_tot = w->gvcf ? w->gv_tot.as<int64_t>() : nullptr;
        A.tile_cov = w->tile_cov.as<int32_t>();
        A.g_meta = w->g_meta.as<uint32_t>(); A.g_read = w->g_read.as<uint32_t>(); A.g_qpos = w->g_qpos.as<uint32_t>();
        A.g_cnt = w->g_cnt.as<uint32_t>(); A.g_next = w->g_next.as<int32_t>(); A.g_used = g_used; A.status = status;
        A.al_meta = w->alleles ? w->al_meta.as<uint32_t>() : nullptr; A.al_read = w->al_read.as<uint32_t>(); A.al_qpos = w->al_qpos.as<uint32_t>();
        A.al_cnt = w->al_cnt.as<uint32_t>(); A.al_off = w->al_off.as<int32_t>(); A.al_n = w->al_n.as<int32_t>();
        A.ins_last = w->ins_last.as<int32_t>(); A.al_used = al_used; A.al_cap = AL_CAP;
        const size_t smem = (size_t)NCNT * TILE * 4 + (size_t)NP * 20;
        plp_count_tile_kernel<<<tiles, TILE, smem, s>>>(A);
        plp_scan_tiles_kernel<<<1, 1024, 0, s>>>(w->tile_cov.as<int32_t>(), w->tile_off.as<int64_t>(), tiles, n_cols_dev);
        EmitArgs E;
        E.start = start; E.end = end; E.call_ht = params->call_ht;
        E.rows32 = w->rows32.as<int32_t>(); E.dstats = w->dstats.as<int32_t>(); E.tile_off = w->tile_off.as<int64_t>();
        E.matrix = w->matrix.as<int64_t>(); E.major = w->major.as<int64_t>(); E.stats = w->stats.as<int32_t>();
        E.dci = w->dci.as<int32_t>(); E.tile_cand = w->tile_cand.as<int32_t>();
        plp_emit_kernel<<<tiles, TILE, 0, s>>>(E);
        plp_quirk_kernel<<<(unsigned)((W + 255) / 256), 256, 0, s>>>(n_cols_dev, w->major.as<int64_t>(), w->nquirk.as<int32_t>(), start,
                                                                      w->matrix.as<int64_t>(), w->stats.as<int32_t>());
        plp_scan_tiles_kernel<<<1, 1024, 0, s>>>(w->tile_cand.as<int32_t>(), w->tile_coff.as<int64_t>(), tiles, n_cand_dev);
        CandArgs C;
        C.start = start; C.end = end; C.n_cols_dev = n_cols_dev; C.dci = w->dci.as<int32_t>(); C.stats = w->stats.as<int32_t>();
        C.major = w->major.as<int64_t>(); C.tile_coff = w->tile_coff.as<int64_t>(); C.cand_cols = w->cand_cols.as<int64_t>();
        C.wstart = w->wstart.as<int64_t>(); C.wbounds = w->wbounds.as<int64_t>(); C.cand_ok = w->cand_ok.as<uint8_t>();
        C.call_ht = params->call_ht;
        plp_cands_kernel<<<tiles, TILE, 0, s>>>(C);
        w->launches += 6;
    }
    C3B_CUDA(cudaEventRecord(w->ev1, s));
    C3B_CUDA(cudaGetLastError());
    C3B_CUDA(cudaMemcpyAsync(w->host_counters, w->counters.p, 32, cudaMemcpyDeviceToHost, s));
    w->counted = true;
    return 0;
}

int c3b_plp_sizes(c3b_plp *w, int64_t *n_cols, int64_t *n_candidates) {
    if (!w || !w->counted) { c3b_set_error("c3b_plp_sizes: no c3b_plp_count has been issued"); return 1; }
    C3B_CUDA(cudaSetDevice(w->device));
    C3B_CUDA(cudaStreamSynchronize(w->stream));
    const int64_t packed = w->host_counters[2];
    const int status = (int)(packed >> 32);
    if (status & 1) { c3b_set_error("c3b_plp_count: more than %d distinct indel alleles spilled from the tiles' shared-memory pools", G_POOL); return 1; }
    if (status & 2) { c3b_set_error("c3b_plp_count: a read spans more than 2^31 reference or query bases"); return 1; }
    if (status & 4) { c3b_set_error("c3b_plp_count: an indel of 2^30 bases or more"); return 1; }
    if (status & 8) { c3b_set_error("c3b_plp_count: more than %d allele records to export (params.alt_info); count a smaller region", AL_CAP); return 1; }
    w->n_cols = w->host_counters[0];
    w->n_cand = w->host_counters[1];
    if (n_cols) *n_cols = w->n_cols;
    if (n_candidates) *n_candidates = w->n_cand;
    return 0;
}

int c3b_plp_fetch(c3b_plp *w, int64_t *matrix, int64_t *major, int32_t *stats, int64_t *cand_cols, uint8_t *cand_ok,
                  int64_t *pos_ref_count, int64_t *pos_total_count) {
    if (!w) { c3b_set_error("c3b_plp_fetch: null workspace"); return 1; }
    if (w->n_cols < 0 && c3b_plp_sizes(w, nullptr, nullptr)) return 1;
    cudaStream_t s = w->stream;
    const size_t nc = (size_t)w->n_cols, nk = (size_t)w->n_cand;
    if (matrix && nc) C3B_CUDA(cudaMemcpyAsync(matrix, w->matrix.p, nc * NFEAT * 8, cudaMemcpyDeviceToHost, s));
    if (major && nc) C3B_CUDA(cudaMemcpyAsync(major, w->major.p, nc * 8, cudaMemcpyDeviceToHost, s));
    if (stats && nc) C3B_CUDA(cudaMemcpyAsync(stats, w->stats.p, nc * 6 * 4, cudaMemcpyDeviceToHost, s));
    if (cand_cols && nk) C3B_CUDA(cudaMemcpyAsync(cand_cols, w->cand_cols.p, nk * 8, cudaMemcpyDeviceToHost, s));
    if (cand_ok && nk) C3B_CUDA(cudaMemcpyAsync(cand_ok, w->cand_ok.p, nk, cudaMemcpyDeviceToHost, s));
    if ((pos_ref_count || pos_total_count) && !w->gvcf) { c3b_set_error("c3b_plp_fetch: the count ran without params.gvcf"); return 1; }
    if (pos_ref_count && w->W) C3B_CUDA(cudaMemcpyAsync(pos_ref_count, w->gv_ref.p, (size_t)w->W * 8, cudaMemcpyDeviceToHost, s));
    if (pos_total_count && w->W) C3B_CUDA(cudaMemcpyAsync(pos_total_count, w->gv_tot.p, (size_t)w->W * 8, cudaMemcpyDeviceToHost, s));
    C3B_CUDA(cudaStreamSynchronize(s));
    return 0;
}

int c3b_plp_fetch_alleles(c3b_plp *w, int32_t *al_off, int32_t *al_n, int32_t *ins_last, uint32_t *meta, uint32_t *read, uint32_t *qpos, uint32_t *cnt,
                          int64_t capacity, int64_t *n_alleles) {
    if (!w) { c3b_set_error("c3b_plp_fetch_alleles: null workspace"); return 1; }
    if (w->n_cols < 0 && c3b_plp_sizes(w, nullptr, nullptr)) return 1;
    if (!w->alleles) { c3b_set_error("c3b_plp_fetch_alleles: the count ran without params.alt_info"); return 1; }
    const int64_t n = (int64_t)(int)(w->host_counters[3] & 0xffffffffll);
    if (n_alleles) *n_alleles = n;
    cudaStream_t s = w->stream;
    if (al_off && w->W) C3B_CUDA(cudaMemcpyAsync(al_off, w->al_off.p, (size_t)w->W * 4, cudaMemcpyDeviceToHost, s));
    if (al_n && w->W) C3B_CUDA(cudaMemcpyAsync(al_n, w->al_n.p, (size_t)w->W * 4, cudaMemcpyDeviceToHost, s));
    if (ins_last && w->W) C3B_CUDA(cudaMemcpyAsync(ins_last, w->ins_last.p, (size_t)w->W * 4, cudaMemcpyDeviceToHost, s));
    if (meta || read || qpos || cnt) {
        if (capacity < n) { c3b_set_error("c3b_plp_fetch_alleles: capacity %lld < %lld records", (long long)capacity, (long long)n); return 1; }
        if (n) {
            if (meta) C3B_CUDA(cudaMemcpyAsync(meta, w->al_meta.p, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
            if (read) C3B_CUDA(cudaMemcpyAsync(read, w->al_read.p, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
            if (qpos) C3B_CUDA(cudaMemcpyAsync(qpos, w->al_qpos.p, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
            if (cnt) C3B_CUDA(cudaMemcpyAsync(cnt, w->al_cnt.p, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
        }
    }
    C3B_CUDA(cudaStreamSynchronize(s));
    return 0;
}

int c3b_plp_device(c3b_plp *w, const int64_t **matrix, const int64_t **major, const int64_t **cand_cols,
                   const int64_t **window_starts, const uint8_t **cand_ok) {
    if (!w || !w->counted) { c3b_set_error("c3b_plp_device: no c3b_plp_count has been issued"); return 1; }
    if (matrix) *matrix = w->matrix.as<int64_t>();
    if (major) *major = w->major.as<int64_t>();
    if (cand_cols) *cand_cols = w->cand_cols.as<int64_t>();
    if (window_starts) *window_starts = w->wstart.as<int64_t>();
    if (cand_ok) *cand_ok = w->cand_ok.as<uint8_t>();
    return 0;
}

int c3b_plp_window_bounds(c3b_plp *w, int64_t *bounds, const int64_t **device_bounds) {
    if (!w) { c3b_set_error("c3b_plp_window_bounds: null workspace"); return 1; }
    if (device_bounds) {
        if (!w->counted) { c3b_set_error("c3b_plp_window_bounds: no c3b_plp_count has been issued"); return 1; }
        *device_bounds = w->wbounds.as<int64_t>();
    }
    if (bounds) {
        if (w->n_cols < 0 && c3b_plp_sizes(w, nullptr, nullptr)) return 1;
        if (w->n_cand) C3B_CUDA(cudaMemcpyAsync(bounds, w->wbounds.p, (size_t)w->n_cand * 16, cudaMemcpyDeviceToHost, w->stream));
        C3B_CUDA(cudaStreamSynchronize(w->stream));
    }
    return 0;
}

int c3b_plp_last_ms(c3b_plp *w, float *ms, int *launches) {
    if (!w || !w->counted) { c3b_set_error("c3b_plp_last_ms: no c3b_plp_count has been issued"); return 1; }
    C3B_CUDA(cudaSetDevice(w->device));
    C3B_CUDA(cudaEventSynchronize(w->ev1));
    float t = 0.f;
    C3B_CUDA(cudaEventElapsedTime(&t, w->ev0, w->ev1));
    if (ms) *ms = t;
    if (launches) *launches = w->launches;
    return 0;
}

void c3b_plp_destroy(c3b_plp *w) {
    if (!w) return;
    cudaSetDevice(w->device);
    DBuf *all[] = {&w->in_pos, &w->in_flag, &w->in_mapq, &w->in_coff, &w->in_cigar, &w->in_soff, &w->in_seq, &w->in_lq, &w->in_ref,
                   &w->opx, &w->opy, &w->rend, &w->pmax, &w->rows32, &w->dstats, &w->nquirk, &w->dci, &w->tile_cov, &w->tile_off,
                   &w->tile_cand, &w->tile_coff, &w->g_meta, &w->g_read, &w->g_qpos, &w->g_cnt, &w->g_next, &w->counters,
                   &w->matrix, &w->major, &w->stats, &w->cand_cols, &w->wstart, &w->wbounds, &w->cand_ok, &w->gv_ref, &w->gv_tot,
                   &w->al_meta, &w->al_read, &w->al_qpos, &w->al_cnt, &w->al_off, &w->al_n, &w->ins_last};
    for (DBuf *b : all) b->release();
    if (w->ev0) cudaEventDestroy(w->ev0);
    if (w->ev1) cudaEventDestroy(w->ev1);
    if (w->host_counters) cudaFreeHost(w->host_counters);
    delete w;
}

}  // extern "C"
