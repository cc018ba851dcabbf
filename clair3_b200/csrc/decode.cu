// First, fully data-parallel stage of the reference's per-site decoder (`batch_output` -> `output_with` -> `output_from` ->
// `possible_outcome_probabilites_from`, clair3/CallVariants.py:1069-1116, 676-700, 510-576) on the GPU, so that only the sites
// that are NOT an early-out homozygous-reference call travel back to the (pure-Python, per-site) decoder:
//   * head slicing gt21 | genotype | indel_1 | indel_2 (param.label_shape_cum, CallVariants.py:1072,1082)
//   * the early-out test  homo_reference >= 0.5 and gt21[ref_base+ref_base] >= 0.5 (and, with indel heads, both
//     variant_length[0 + index_offset] >= 0.5)                                   CallVariants.py:532-534, 573-576
//   * homo_Ref_probability, the product the early-out returns, in the reference's float32 evaluation order   :527, 569-572
//   * per-head arg-max (first maximum, like numpy) and max probability
//   * QUAL of the early-out call, quality_score_from before its round(.., 2)       CallVariants.py:375-381
//   * the stable (ascending) compaction of the remaining site indices.
// Integer outputs (flags, arg-max, indices, count) are bit-exact vs the numpy restatement in oracle/decode_oracle.py; the
// float32 product is IEEE-exact (no contraction: multiplies only).
#include "c3b_internal.h"

#include <algorithm>
#include <climits>

namespace {

constexpr int kDecodeThreads = 1024;

struct DecodeDev {
    const float *y;
    const uint8_t *ref_gt21;
    int64_t batch;
    int out_dim, nheads;
    uint8_t *is_ref;
    float *ref_prob;
    int32_t *argmax;      // [batch][nheads]
    float *maxprob;       // [batch][nheads]
    double *qual;         // [batch]
    int32_t *nonref_idx;  // [batch]
    int32_t *n_nonref;    // [1]
};

__global__ void __launch_bounds__(kDecodeThreads) decode_stage1_kernel(const DecodeDev p) {
    __shared__ int warp_cnt[32];
    __shared__ int base_s;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int off[5] = {0, 21, 24, 57, 90};
    if (tid == 0) base_s = 0;
    __syncthreads();
    for (int64_t b0 = 0; b0 < p.batch; b0 += kDecodeThreads) {
        const int64_t b = b0 + tid;
        bool nonref = false;
        if (b < p.batch) {
            const float *row = p.y + b * p.out_dim;
            for (int h = 0; h < p.nheads; ++h) {
                int am = 0;
                float mx = row[off[h]];
                for (int o = off[h] + 1; o < off[h + 1]; ++o) {
                    const float v = row[o];
                    if (v > mx) { mx = v; am = o - off[h]; }
                }
                p.argmax[b * p.nheads + h] = am;
                p.maxprob[b * p.nheads + h] = mx;
            }
            const float homo_ref = row[21 + 0];                       // Genotype.homo_reference = 0 (clair3/task/genotype.py:7)
            const float gt_ref = row[p.ref_gt21[b]];
            bool early = homo_ref >= 0.5f && gt_ref >= 0.5f;
            float prob;
            if (p.nheads == 4) {
                const float v1 = row[24 + 16], v2 = row[57 + 16];     // variant_length index_offset = 16 (task/variant_length.py:6)
                early = early && v1 >= 0.5f && v2 >= 0.5f;
                prob = __fmul_rn(__fmul_rn(__fmul_rn(v1, v2), homo_ref), gt_ref);
            } else {
                prob = __fmul_rn(homo_ref, gt_ref);
            }
            p.is_ref[b] = early ? 1 : 0;
            p.ref_prob[b] = prob;
            // quality_score_from: max(Phred_Trans * log(((1.0 - p) + 1e-10) / (p + 1e-10)) + 10, 0); the ratio is float32 arithmetic
            // on a numpy float32 scalar (NumPy >= 2 promotion), the log is math.log of that value in double
            const float ratio = __fdiv_rn(__fadd_rn(__fsub_rn(1.0f, prob), 1e-10f), __fadd_rn(prob, 1e-10f));
            const double q = -4.342944819032518 * log((double)ratio) + 10.0;
            p.qual[b] = q > 0.0 ? q : 0.0;
            nonref = !early;
        }
        // stable compaction of the non-reference sites of this 1024-site slab
        const unsigned bal = __ballot_sync(0xffffffffu, nonref);
        if (lane == 0) warp_cnt[warp] = __popc(bal);
        __syncthreads();
        int before = 0, total = 0;
        for (int w = 0; w < 32; ++w) {
            const int c = warp_cnt[w];
            if (w < warp) before += c;
            total += c;
        }
        if (nonref) p.nonref_idx[base_s + before + __popc(bal & ((1u << lane) - 1u))] = (int32_t)b;
        __syncthreads();
        if (tid == 0) base_s += total;
        __syncthreads();
    }
    if (tid == 0) *p.n_nonref = base_s;
}

}  // namespace

int c3b_launch_decode_stage1(const float *y, const uint8_t *ref_gt21, int64_t batch, int out_dim, uint8_t *is_ref, float *ref_prob,
                             int32_t *argmax, float *maxprob, double *qual, int32_t *nonref_idx, int32_t *n_nonref, cudaStream_t s) {
    DecodeDev p;
    p.y = y; p.ref_gt21 = ref_gt21; p.batch = batch; p.out_dim = out_dim; p.nheads = out_dim == 90 ? 4 : 2;
    p.is_ref = is_ref; p.ref_prob = ref_prob; p.argmax = argmax; p.maxprob = maxprob; p.qual = qual;
    p.nonref_idx = nonref_idx; p.n_nonref = n_nonref;
    decode_stage1_kernel<<<1, kDecodeThreads, 0, s>>>(p);
    C3B_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------ stage 2
// Second stage: for every listed site, the outcome lists possible_outcome_probabilites_from builds (CallVariants.py:413-494 with
// the indel-length heads, :519-562 without: 804 or 24 float32 products, multiplies only, the reference's left-to-right order)
// and the order in which output_from (:720-1005) tries them: probability descending, then category in output_from's elif order
// (homo_Ref first), then index within the category's list.  The first k entries of that order, ending at homo_Ref, are
// emitted with their tie mask: bit c = category c holds an entry of the same probability at this position or later, which is
// the is_* flag tuple output_from returns when this attempt succeeds.  Restated in oracle/decode_stage2_oracle.py.
//
// One warp per site.  Slot e (the lists concatenated in category order) lives in lane e % 32, register e / 32, as the bits of
// its non-negative float (-1 once emitted); every lane keeps its best (bits, -slot) key, and each round is one 64-bit warp max.
namespace {

constexpr int kStage2Warps = 8;

struct Stage2Dev {
    const float *y;
    const uint8_t *ref_gt21;
    int64_t batch;
    const int32_t *sites;     // null: site s is row s
    const int32_t *n_sites;   // null: max_sites
    int64_t max_sites;
    int k;
    uint8_t *cat;
    uint16_t *idx;
    float *prob;
    uint16_t *tie_mask;
    int32_t *count;
    uint8_t *complete;
};

// first slot of each category, and one past the last
__constant__ int kStart90[11] = {0, 1, 5, 11, 27, 91, 227, 243, 307, 548, 804};
__constant__ int kStart24[11] = {0, 1, 5, 11, 12, 16, 17, 18, 22, 23, 24};

template <int OUT>
__device__ __forceinline__ int slot_category(int e) {
    int c = 0;
#pragma unroll
    for (int i = 1; i < 10; ++i) c += e >= (OUT == 90 ? kStart90[i] : kStart24[i]);
    return c;
}

__device__ __forceinline__ float fm(float a, float b) { return __fmul_rn(a, b); }

// gt21 columns: AA 0 AC 1 AG 2 AT 3 CC 4 CG 5 CT 6 GG 7 GT 8 TT 9 DelDel 10 ADel..TDel 11-14 InsIns 15 AIns..TIns 16-19 InsDel 20
__device__ __forceinline__ int homo_snp_col(int j) { return j == 0 ? 0 : j == 1 ? 4 : j == 2 ? 7 : 9; }
__device__ __forceinline__ int hetero_snp_col(int j) { return j < 3 ? j + 1 : j == 3 ? 5 : j == 4 ? 6 : 8; }

__device__ float slot_value90(int e, const float *r, float gref) {
    const float *g = r, *v1 = r + 24, *v2 = r + 57;
    const float homref = r[21], homvar = r[22], hetvar = r[23];
    const float vl0 = fm(v1[16], v2[16]);
    if (e == 0) return fm(fm(vl0, homref), gref);
    if (e < 5) return fm(fm(vl0, homvar), g[homo_snp_col(e - 1)]);
    if (e < 11) return fm(fm(vl0, hetvar), g[hetero_snp_col(e - 5)]);
    if (e < 27) { const int i = e - 11 + 1; return fm(fm(v1[16 + i], v2[16 + i]), fm(homvar, g[15])); }
    if (e < 91) { const int j = e - 27, i = j / 4 + 1; return fm(fm(fm(v1[16], v2[16 + i]), g[16 + j % 4]), hetvar); }
    if (e < 227) {                                   // i <= j, i outer
        int j = e - 91, i = 1;
        while (j >= 17 - i) { j -= 17 - i; ++i; }
        return fm(fm(v1[16 + i], v2[16 + i + j]), fm(hetvar, g[15]));
    }
    if (e < 243) { const int i = e - 227 + 1; return fm(fm(v1[16 - i], v2[16 - i]), fm(homvar, g[10])); }
    if (e < 307) { const int j = e - 243, i = j / 4 + 1; return fm(fm(fm(v1[16 - i], v2[16]), g[11 + j % 4]), hetvar); }
    if (e < 548) {                                   // 16 x 16 without i == j != 16, i outer: rows 1..15 hold 15, row 16 holds 16
        const int q = e - 307;
        int i, j;
        if (q < 225) { i = q / 15 + 1; j = q % 15 + 1; j += j >= i; }
        else { i = 16; j = q - 225 + 1; }
        return fm(fm(v1[16 - i], v2[16 - j]), fm(hetvar, g[10]));
    }
    const int q = e - 548, i = q / 16 + 1, j = q % 16 + 1;
    return fm(fm(v1[16 - i], v2[16 + j]), fm(hetvar, g[20]));
}

__device__ float slot_value24(int e, const float *g, float gref) {
    const float homref = g[21], homvar = g[22], hetvar = g[23];
    if (e == 0) return fm(homref, gref);
    if (e < 5) return fm(homvar, g[homo_snp_col(e - 1)]);
    if (e < 11) return fm(hetvar, g[hetero_snp_col(e - 5)]);
    if (e == 11) return fm(homvar, g[15]);
    if (e < 16) return fm(g[16 + e - 12], hetvar);
    if (e == 16) return fm(hetvar, g[15]);
    if (e == 17) return fm(homvar, g[10]);
    if (e < 22) return fm(g[11 + e - 18], hetvar);
    if (e == 22) return fm(hetvar, g[10]);
    return fm(hetvar, g[20]);
}

template <int OUT>
__global__ void __launch_bounds__(kStage2Warps * 32) decode_stage2_kernel(const Stage2Dev p) {
    constexpr int E = OUT == 90 ? 804 : 24;
    constexpr int NJ = (E + 31) / 32;
    __shared__ float rows[kStage2Warps][96];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    int64_t n = p.max_sites;
    if (p.n_sites) n = max((int64_t)0, min((int64_t)*p.n_sites, p.max_sites));
    float *row = rows[wib];
    for (int64_t s = (int64_t)blockIdx.x * kStage2Warps + wib; s < p.max_sites; s += (int64_t)gridDim.x * kStage2Warps) {
        const int64_t site = s < n ? (p.sites ? (int64_t)p.sites[s] : s) : -1;
        int cnt = 0;
        bool done = false;
        if (site >= 0 && site < p.batch) {
            __syncwarp();
            for (int o = lane; o < OUT; o += 32) row[o] = p.y[site * OUT + o];
            __syncwarp();
            const float gref = row[p.ref_gt21[site]];
            int key[NJ];
#pragma unroll
            for (int j = 0; j < NJ; ++j) {
                const int e = j * 32 + lane;
                key[j] = e < E ? __float_as_int(OUT == 90 ? slot_value90(e, row, gref) : slot_value24(e, row, gref)) : -1;
            }
            auto local_best = [&]() {
                long long b = LLONG_MIN;
#pragma unroll
                for (int j = 0; j < NJ; ++j) {
                    const long long c = ((long long)key[j] << 32) | (long long)(0xFFFF - (j * 32 + lane));
                    b = c > b ? c : b;
                }
                return b;
            };
            long long mine = local_best();
            const int64_t base = s * p.k;
            for (int t = 0; t < p.k; ++t) {
                long long w = mine;
#pragma unroll
                for (int o = 16; o; o >>= 1) {
                    const long long x = __shfl_xor_sync(0xffffffffu, w, o);
                    w = x > w ? x : w;
                }
                const int wbits = (int)(w >> 32);
                const int e = 0xFFFF - (int)(w & 0xFFFF);
                unsigned m = 0;
#pragma unroll
                for (int j = 0; j < NJ; ++j)
                    if (key[j] == wbits) m |= 1u << slot_category<OUT>(j * 32 + lane);
                m = __reduce_or_sync(0xffffffffu, m);
                if (lane == 0) {
                    const int c = slot_category<OUT>(e);
                    p.cat[base + t] = (uint8_t)c;
                    p.idx[base + t] = (uint16_t)(e - (OUT == 90 ? kStart90[c] : kStart24[c]));
                    p.prob[base + t] = __int_as_float(wbits);
                    p.tie_mask[base + t] = (uint16_t)m;
                }
                if (lane == (e & 31)) {
#pragma unroll
                    for (int j = 0; j < NJ; ++j)
                        if (j == (e >> 5)) key[j] = -1;
                    mine = local_best();
                }
                cnt = t + 1;
                if (e == 0) { done = true; break; }   // homo_Ref: output_from returns a reference call here at the latest
            }
        }
        for (int t = cnt + lane; t < p.k; t += 32) {
            p.cat[s * p.k + t] = 255;
            p.idx[s * p.k + t] = 0;
            p.prob[s * p.k + t] = 0.0f;
            p.tie_mask[s * p.k + t] = 0;
        }
        if (lane == 0) {
            p.count[s] = cnt;
            p.complete[s] = done ? 1 : 0;
        }
    }
}

}  // namespace

int c3b_launch_decode_stage2(const float *y, const uint8_t *ref_gt21, int64_t batch, int out_dim, const int32_t *sites,
                             const int32_t *n_sites, int64_t max_sites, int k, uint8_t *cat, uint16_t *idx, float *prob,
                             uint16_t *tie_mask, int32_t *count, uint8_t *complete, cudaStream_t s) {
    if (max_sites <= 0) return 0;
    Stage2Dev p;
    p.y = y; p.ref_gt21 = ref_gt21; p.batch = batch; p.sites = sites; p.n_sites = n_sites; p.max_sites = max_sites; p.k = k;
    p.cat = cat; p.idx = idx; p.prob = prob; p.tie_mask = tie_mask; p.count = count; p.complete = complete;
    const int64_t blocks = std::min<int64_t>((max_sites + kStage2Warps - 1) / kStage2Warps, 8192);
    if (out_dim == 90) decode_stage2_kernel<90><<<(unsigned)blocks, kStage2Warps * 32, 0, s>>>(p);
    else decode_stage2_kernel<24><<<(unsigned)blocks, kStage2Warps * 32, 0, s>>>(p);
    C3B_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------ stage 3: the calls
// Third stage: walks every listed site's ranked entries (stage 2's output) against its alt_info and fills the c3b_call record
// (clair3_b200.h).  The statement is clair3_b200/decode.py: parse_alt_info, _try_outcome and its helpers, output_from_ranked,
// and format_row's filters, genotype, DP, AD and AF support.  Restated on the host in oracle/decode_calls_oracle.py.
//
// One warp per site.  Lane 0 tokenises the alt_info string into the site's allele table (global scratch, alt_offsets[s] + s,
// len + 1 entries) and the warp merges repeated keys as dict(zip()) does; keys are then unique, so every string test of the host code on a key becomes an
// allele-index test.  Every lane then runs the same walk: each selection is one warp arg-max over the alleles (lane a % 32
// scans allele a) of a predicate with a (count, +-index) key; a string the walk has built (REF / ALT in the site's text region)
// is compared byte for byte where format_row looks it up.
namespace {

constexpr int kCallWarps = 4;
constexpr long long kNone = LLONG_MIN;
constexpr long long kCountMax = 1LL << 62;

struct CallAllele {
    int64_t start;      // first byte of the key in alt_bytes
    int32_t len;        // key length (kind byte included)
    int32_t last;       // while merging repeated keys: the key's last token (-1: not its first token)
    uint8_t kind, b1;   // key[0], key[1] (0 when absent)
    long long count;
};

struct CallsDev {
    const char *bytes;
    const int64_t *off;
    int64_t n_bytes;
    const uint8_t *ref_base;
    int64_t batch;
    int add_indel;
    uint32_t cfg;
    long long max_len;
    const uint8_t *is_ref;     // stage 1; null: no early-out rows in this pass
    const float *ref_prob;
    const int32_t *sites;      // listed sites and their ranked rows (row r = stage 2's row r)
    const int32_t *n_sites;
    int64_t max_rows;
    int k;
    const uint8_t *cat;
    const uint16_t *idx;
    const float *prob;
    const uint16_t *tie;
    const int32_t *count;
    CallAllele *tab;
    uint8_t *unresolved;       // [batch] set where the k entries run out
    c3b_call *calls;
    char *text;
    long long *ad;
};

__device__ __forceinline__ bool py_space(unsigned char c) { return c == ' ' || (c >= 9 && c <= 13) || (c >= 0x1c && c <= 0x1f); }

// Python's int() on an ASCII token: 0 ok, 1 ValueError, 4 out of +-2^62
__device__ int py_int(const char *s, int64_t n, long long *v) {
    int64_t a = 0, b = n;
    while (a < b && py_space(s[a])) ++a;
    while (b > a && py_space(s[b - 1])) --b;
    bool neg = false;
    if (a < b && (s[a] == '+' || s[a] == '-')) { neg = s[a] == '-'; ++a; }
    if (a >= b) return 1;
    long long x = 0;
    bool digit = false, big = false;
    for (int64_t i = a; i < b; ++i) {
        const char c = s[i];
        if (c == '_') {
            if (!digit) return 1;
            digit = false;
            continue;
        }
        if (c < '0' || c > '9') return 1;
        if (!big) {
            big = x > (kCountMax - (c - '0')) / 10;           // before the multiply: x * 10 + d must stay <= 2^62
            if (!big) x = x * 10 + (c - '0');
        }
        digit = true;
    }
    if (!digit) return 1;
    if (big) return 4;
    *v = neg ? -x : x;
    return 0;
}

__device__ __forceinline__ int acgt_of(unsigned char c) {       // IUPAC_base_to_ACGT_base_dict, 0 = not a key
    switch (c) {
        case 'A': case 'R': case 'W': case 'M': case 'D': case 'H': case 'V': case 'N': return 'A';
        case 'C': case 'Y': case 'S': case 'B': return 'C';
        case 'G': case 'K': return 'G';
        case 'T': case 'U': return 'T';
        default: return 0;
    }
}

// warp arg-max of key(a) over alleles [0, n); kNone = not a candidate; ties: lowest index (low) or highest.  -1: none
template <class Key>
__device__ int warp_best(int n, bool low, Key key, long long *best = nullptr) {
    const int lane = threadIdx.x & 31;
    long long c = kNone;
    int i = -1;
    for (int a = lane; a < n; a += 32) {
        const long long v = key(a);
        if (v != kNone && (i < 0 || v > c || (v == c && !low))) { c = v; i = a; }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const long long oc = __shfl_xor_sync(0xffffffffu, c, o);
        const int oi = __shfl_xor_sync(0xffffffffu, i, o);
        const bool take = oi >= 0 && (i < 0 || oc > c || (oc == c && (low ? oi < i : oi > i)));
        if (take) { c = oc; i = oi; }
    }
    if (best) *best = c;
    return i;
}

template <class F>
__device__ long long warp_sum(int n, F f) {
    long long s = 0;
    for (int a = threadIdx.x & 31; a < n; a += 32) s += f(a);
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    return s;
}

__device__ __forceinline__ bool same_bytes(const char *a, const char *b, int n) {
    for (int i = 0; i < n; ++i)
        if (a[i] != b[i]) return false;
    return true;
}

// one piece of an allele text: pre (0: none), then allele a1's bases (key[1:]) from byte skip on, then allele a2's bases
struct Piece { char pre; int a1, skip, a2; };

struct Site {
    const CallsDev *p;
    const CallAllele *t;
    int n;                     // alleles
    bool bad_empty, bad_x;     // an empty key / a bare "X" key: indexing them raises IndexError
    char r;                    // raw reference base
    __device__ int blen(int a) const { return t[a].len - 1; }
    __device__ const char *bases(int a) const { return p->bytes + t[a].start + 1; }
    __device__ int piece_len(const Piece &q) const {
        return (q.pre ? 1 : 0) + (q.a1 >= 0 ? blen(q.a1) - q.skip : 0) + (q.a2 >= 0 ? blen(q.a2) : 0);
    }
    // _indel_bases: the best allele of `kind` of length `prop` (0: no proposal), else within [1, max_len]; never `ignore`
    __device__ int indel(char kind, int prop, int ignore) const {
        if (n == 0) return -1;
        const long long ml = p->max_len;
        if (prop) {
            const int a = warp_best(n, true, [&](int a) {
                return t[a].kind == kind && blen(a) == prop && a != ignore ? t[a].count : kNone; });
            if (a >= 0) return a;
        }
        return warp_best(n, true, [&](int a) {
            return t[a].kind == kind && blen(a) >= 1 && blen(a) <= ml && a != ignore ? t[a].count : kNone; });
    }
    // return_multi: the two best, sorted ascending (stable) then reversed - equal counts: the later allele first
    __device__ int multi(char kind, int *second) const {
        const long long ml = p->max_len;
        auto ok = [&](int a) { return t[a].kind == kind && blen(a) >= 1 && blen(a) <= ml; };
        const int a0 = n ? warp_best(n, false, [&](int a) { return ok(a) ? t[a].count : kNone; }) : -1;
        *second = a0 < 0 ? -1 : warp_best(n, false, [&](int a) { return ok(a) && a != a0 ? t[a].count : kNone; });
        return a0;
    }
    __device__ int ins(int length, int ignore = -1) const { return indel('I', length > 0 && length < 16 ? length + 1 : 0, ignore); }
    __device__ int del(int length, int ignore = -1) const { return indel('D', length > 0 && length < 16 ? length : 0, ignore); }
    // find_alt_base: the best SNP allele (first maximum); with a proposed base, that base unless absent or 9+ reads behind
    __device__ char alt_base(char proposed) const {
        long long cb;
        const int b = warp_best(n, true, [&](int a) { return t[a].kind == 'X' ? t[a].count : kNone; }, &cb);
        if (b < 0) return 0;
        long long cp;
        const int q = warp_best(n, true, [&](int a) { return t[a].kind == 'X' && t[a].b1 == (uint8_t)proposed ? t[a].count : kNone; }, &cp);
        return q < 0 || cb - cp >= 9 ? (char)t[b].b1 : proposed;
    }
};

__constant__ char kHomoSnp[4][2] = {{'A', 'A'}, {'C', 'C'}, {'G', 'G'}, {'T', 'T'}};
__constant__ char kHeteroSnp[6][2] = {{'A', 'C'}, {'A', 'G'}, {'A', 'T'}, {'C', 'G'}, {'C', 'T'}, {'G', 'T'}};
__device__ __forceinline__ char acgt(int i) { return i == 0 ? 'A' : i == 1 ? 'C' : i == 2 ? 'G' : 'T'; }

struct Outcome {
    int del;          // REF = r + allele del's bases (-1: r alone)
    int np;           // ALT pieces, joined by ','
    Piece q[2];
};

__device__ __forceinline__ Piece pc(char pre, int a1 = -1, int skip = 0, int a2 = -1) { Piece q; q.pre = pre; q.a1 = a1; q.skip = skip; q.a2 = a2; return q; }

// _try_outcome: 1 success (o filled), 0 the reads do not support it, 2 IndexError (a helper indexed a bad key)
__device__ int try_outcome(const Site &S, int cat, int idx, Outcome &o) {
    const bool add = S.p->add_indel;
    const char r = S.r;
    const bool snp_err = S.bad_empty || S.bad_x, indel_err = S.bad_empty;
    o.del = -1;
    o.np = 1;
    switch (cat) {
        case 1: case 2: {
            const char b1 = cat == 1 ? kHomoSnp[idx][0] : kHeteroSnp[idx][0], b2 = cat == 1 ? kHomoSnp[idx][1] : kHeteroSnp[idx][1];
            if (snp_err) return 2;
            if (cat == 2 && b1 != r && b2 != r) {
                const int a0 = warp_best(S.n, true, [&](int a) { return S.t[a].kind == 'X' ? S.t[a].count : kNone; });
                const int a1 = a0 < 0 ? -1 : warp_best(S.n, true, [&](int a) { return S.t[a].kind == 'X' && a != a0 ? S.t[a].count : kNone; });
                if (a1 < 0) return 0;
                o.np = 2;
                o.q[0] = pc((char)S.t[a0].b1);
                o.q[1] = pc((char)S.t[a1].b1);
                return 1;
            }
            const char alt = S.alt_base(b1 != r ? b1 : b2);
            if (!alt) return 0;
            o.q[0] = pc(alt);
            return 1;
        }
        case 3: {
            if (indel_err) return 2;
            const int a = S.ins(add ? idx + 1 : 0);
            if (a < 0) return 0;
            o.q[0] = pc(0, a);
            return 1;
        }
        case 4: {
            const char base = add ? acgt(idx % 4) : acgt(idx);
            if (indel_err) return 2;
            const int a = S.ins(add ? idx / 4 + 1 : 0);
            if (a < 0) return 0;
            if (base != r) {
                if (snp_err) return 2;
                const int s = warp_best(S.n, true, [&](int x) { return S.t[x].kind == 'X' ? S.t[x].count : kNone; });
                if (s >= 0) {
                    o.np = 2;
                    o.q[0] = pc((char)S.t[s].b1);
                    o.q[1] = pc(0, a);
                    return 1;
                }
            }
            o.q[0] = pc(0, a);
            return 1;
        }
        case 5: {
            if (indel_err) return 2;
            int p0 = -1, p1 = -1;
            if (add) {
                int l1 = 1, j = idx;                       // INSINS_PAIRS: (i, j), i <= j, i outer
                while (j >= 17 - l1) { j -= 17 - l1; ++l1; }
                const int l2 = l1 + j;
                const int b1 = S.ins(l1);
                if (b1 >= 0) {
                    const int b2 = S.ins(l2, b1);
                    if (b2 >= 0) { p0 = b1; p1 = b2; }
                }
            }
            if (p1 < 0) p0 = S.multi('I', &p1);
            if (p1 < 0) return 0;
            o.np = 2;
            o.q[0] = pc(0, p1);
            o.q[1] = pc(0, p0);
            return 1;
        }
        case 6: case 7: {
            char base = 0;
            int length = 0;
            if (cat == 6) length = add ? idx + 1 : 0;
            else { base = add ? acgt(idx % 4) : acgt(idx); length = add ? idx / 4 + 1 : 0; }
            if (indel_err) return 2;
            const int d = S.del(length);
            if (d < 0) return 0;
            o.del = d;
            if (base && base != r) {
                o.np = 2;
                o.q[0] = pc(r);
                o.q[1] = pc(base, d);
            } else {
                o.q[0] = pc(r);
            }
            return 1;
        }
        case 8: {
            if (indel_err) return 2;
            int p0 = -1, p1 = -1;
            if (add) {
                int i, j;                                  // DELDEL_PAIRS, list order
                if (idx < 225) { i = idx / 15 + 1; j = idx % 15 + 1; j += j >= i; }
                else { i = 16; j = idx - 225 + 1; }
                const int l1 = max(i, j), l2 = min(i, j);
                const int b1 = S.del(l1);
                if (b1 >= 0) {
                    const int b2 = S.del(l2, b1);
                    if (b2 >= 0) {
                        if (S.blen(b1) > S.blen(b2)) { p0 = b1; p1 = b2; } else { p0 = b2; p1 = b1; }
                    }
                }
            }
            if (p1 < 0) {
                int r1;
                const int r0 = S.multi('D', &r1);
                if (r1 < 0) return 0;
                if (S.blen(r0) > S.blen(r1)) { p0 = r0; p1 = r1; } else { p0 = r1; p1 = r0; }
            }
            o.del = p0;
            const int l0 = S.blen(p0), l1 = S.blen(p1);
            if (l0 > l1 && l1 != 0) {
                o.np = 2;
                o.q[0] = pc(r);
                o.q[1] = pc(r, p0, l1);
            } else {
                o.q[0] = pc(r);
            }
            return 1;
        }
        default: {                                         // 9: hetero_InsDel
            const int l_del = add ? idx / 16 + 1 : 0, l_ins = add ? idx % 16 + 1 : 0;
            if (indel_err) return 2;
            const int a = S.ins(l_ins), d = S.del(l_del);
            if (a < 0 || d < 0) return 0;
            o.del = d;
            o.np = 2;
            o.q[0] = pc(r);
            o.q[1] = pc(0, a, 0, d);
            return 1;
        }
    }
}

// warp-cooperative copy of n bytes
__device__ __forceinline__ void wcopy(char *dst, const char *src, int n) {
    for (int i = threadIdx.x & 31; i < n; i += 32) dst[i] = src[i];
}

__device__ int write_piece(const Site &S, char *dst, const Piece &q) {
    int o = 0;
    if (q.pre) { if ((threadIdx.x & 31) == 0) dst[0] = q.pre; o = 1; }
    if (q.a1 >= 0) { const int n = S.blen(q.a1) - q.skip; wcopy(dst + o, S.bases(q.a1) + q.skip, n); o += n; }
    if (q.a2 >= 0) { const int n = S.blen(q.a2); wcopy(dst + o, S.bases(q.a2), n); o += n; }
    return o;
}

// format_row's lookups on text the walk has built
struct Rows {
    const Site &S;
    bool long_indel;
    // snp.get(c, 0): the last SNP key whose key[1] is c
    __device__ long long snp(char c) const {
        const int a = warp_best(S.n, false, [&](int a) { return S.t[a].kind == 'X' && S.t[a].b1 == (uint8_t)c ? 0LL : kNone; });
        return a < 0 ? 0 : S.t[a].count;
    }
    // ins.get(s, 0) / dels.get(s, 0)
    __device__ long long get(char kind, const char *s, int n) const {
        const int a = warp_best(S.n, true, [&](int a) {
            return S.t[a].kind == kind && S.blen(a) == n && same_bytes(S.bases(a), s, n) ? 0LL : kNone; });
        return a < 0 ? 0 : S.t[a].count;
    }
    // _long_indel_reads(ins, proposed_ins_base=s): other insertions within 10 % of the proposed length, from 51 bases on
    __device__ long long long_ins(const char *s, int n) const {
        if (!long_indel || n <= 50) return 0;
        const double length = (double)(n - 1);
        const double lo = fmax(__dmul_rn(length, 1.0 - 0.1), 50.0), hi = __dmul_rn(length, 1.0 + 0.1);
        return warp_sum(S.n, [&](int a) -> long long {
            if (S.t[a].kind != 'I') return 0;
            const int l = S.blen(a);
            if (!(lo <= (double)l && (double)l <= hi)) return 0;
            return l == n && same_bytes(S.bases(a), s, n) ? 0 : S.t[a].count;
        });
    }
    // _deletion_reads: the first deletion of that length
    __device__ long long del_len(long long length) const {
        const int a = warp_best(S.n, true, [&](int a) { return S.t[a].kind == 'D' && S.blen(a) == length ? 0LL : kNone; });
        return a < 0 ? 0 : S.t[a].count;
    }
};

__device__ void decode_site(const CallsDev &p, int64_t site, int64_t row) {
    const int lane = threadIdx.x & 31;
    c3b_call *out = p.calls + site;
    const int64_t s0 = p.off[site], s1 = p.off[site + 1];
    const unsigned char rb = p.ref_base[site];
    if (s0 < 0 || s1 < s0 || s1 > p.n_bytes || !acgt_of(rb)) {
        if (lane == 0) { memset(out, 0, sizeof(c3b_call)); out->status = 5; out->genotype = 255; }
        return;
    }
    const char *a = p.bytes + s0;
    const int64_t cap = 2 * (s1 - s0) + 8;
    char *text = p.text + 2 * s0 + 8 * site;
    long long *ad = p.ad + 2 * s0 + 8 * site;
    CallAllele *tab = p.tab + s0 + site;
    // ---- parse_alt_info (lane 0)
    int status = 0, na = 0, bad = 0;
    long long depth = 0;
    if (lane == 0) {
        int64_t L = s1 - s0;
        for (int64_t i = 0; i < L && !status; ++i)
            if ((unsigned char)a[i] >= 0x80) status = 4;
        while (L > 0 && py_space(a[L - 1])) --L;
        int64_t d1 = 0;
        while (d1 < L && a[d1] != '-') ++d1;
        bool big = false;                                 // a count beyond +-2^62: status 4 unless a token fails to parse
        if (!status) { status = py_int(a, d1, &depth); big = status == 4; status = status == 4 ? 0 : status; }
        int64_t pos = d1 < L ? d1 + 1 : L, be = pos;
        while (be < L && a[be] != '-') ++be;
        int64_t kpos = 0;
        int klen = 0;
        for (int tok = 0; !status; ++tok) {
            int64_t e = pos;
            while (e < be && a[e] != ' ') ++e;
            if (!(tok & 1)) {
                kpos = pos;
                klen = (int)(e - pos);
            } else {
                long long v = 0;
                status = py_int(a + pos, e - pos, &v);
                if (status == 4) { big = true; status = 0; v = 0; }
                if (!status) {
                    CallAllele c;
                    c.start = s0 + kpos;
                    c.len = klen;
                    c.last = -1;
                    c.kind = klen > 0 ? (uint8_t)a[kpos] : 0;
                    c.b1 = klen > 1 ? (uint8_t)a[kpos + 1] : 0;
                    c.count = v;
                    tab[na++] = c;
                }
            }
            if (e >= be) break;
            pos = e + 1;
        }
        if (!status && big) status = 4;
    }
    __syncwarp();
    status = __shfl_sync(0xffffffffu, status, 0);
    if (status) {
        if (lane == 0) { memset(out, 0, sizeof(c3b_call)); out->status = (uint8_t)status; out->genotype = 255; }
        return;
    }
    na = __shfl_sync(0xffffffffu, na, 0);
    depth = __shfl_sync(0xffffffffu, depth, 0);
    // dict(zip(keys, counts)): a repeated key keeps its first token's position and takes its last token's count.  Lane
    // i % 32 finds token i's first and last equal token, then the first tokens are compacted in order.
    auto same_key = [&](int i, int j) {
        return tab[i].len == tab[j].len && same_bytes(p.bytes + tab[i].start, p.bytes + tab[j].start, tab[i].len);
    };
    for (int i = lane; i < na; i += 32) {
        int first = i;
        for (int j = 0; j < i && first == i; ++j)
            if (same_key(i, j)) first = j;
        int last = i;
        if (first == i)
            for (int j = na - 1; j > i && last == i; --j)
                if (same_key(i, j)) last = j;
        tab[i].last = first == i ? last : -1;
    }
    __syncwarp();
    int kept = 0;
    for (int i0 = 0; i0 < na; i0 += 32) {
        const int i = i0 + lane;
        CallAllele c;
        bool keep = false;
        if (i < na) {
            c = tab[i];
            keep = c.last >= 0;
            if (keep) c.count = tab[c.last].count;
        }
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        __syncwarp();
        if (keep) {
            tab[kept + __popc(bal & ((1u << lane) - 1u))] = c;
            bad |= (c.len == 0 ? 1 : 0) | (c.len == 1 && c.kind == 'X' ? 2 : 0);
        }
        kept += __popc(bal);
        __syncwarp();
    }
    na = kept;
    bad = __reduce_or_sync(0xffffffffu, bad);
    Site S;
    S.p = &p; S.t = tab; S.n = na; S.bad_empty = bad & 1; S.bad_x = (bad & 2) != 0; S.r = (char)rb;
    // ---- the walk (output_from_ranked)
    uint16_t flags = 1;
    float prob;
    Outcome o;
    bool is_ref = true;
    if (row < 0) {
        prob = p.ref_prob[site];
    } else {
        const int64_t base = row * p.k;
        const int cnt = p.count[row];
        int got = 0, t = 0;
        for (; t < cnt; ++t) {
            const int c = p.cat[base + t];
            if (c == 0) { got = 3; break; }
            got = try_outcome(S, c, p.idx[base + t], o);
            if (got) break;
        }
        if (got == 0) {                                    // the entries ran out: re-rank this site with the full list
            if (lane == 0) p.unresolved[site] = 1;
            return;
        }
        if (got == 2) {
            if (lane == 0) { memset(out, 0, sizeof(c3b_call)); out->status = 2; out->genotype = 255; }
            return;
        }
        prob = p.prob[base + t];
        if (got == 1) { flags = p.tie[base + t]; is_ref = false; }
    }
    // ---- REF and ALT text as output_from returns them
    const char racgt = (char)acgt_of(rb);
    int ref_len, alt_len;
    if (is_ref) {
        ref_len = alt_len = 1;
    } else {
        ref_len = 1 + (o.del >= 0 ? S.blen(o.del) : 0);
        alt_len = o.np - 1;
        for (int i = 0; i < o.np; ++i) alt_len += S.piece_len(o.q[i]);
    }
    if (ref_len + alt_len > cap) {                       // cannot happen: REF + ALT <= 2 * len(alt_info) + 8
        if (lane == 0) { memset(out, 0, sizeof(c3b_call)); out->status = 4; out->genotype = 255; }
        return;
    }
    char *ref = text, *alt = text + ref_len;
    if (is_ref) {
        if (lane == 0) { ref[0] = racgt; alt[0] = racgt; }
    } else {
        if (lane == 0) ref[0] = S.r;
        if (o.del >= 0) wcopy(ref + 1, S.bases(o.del), S.blen(o.del));
        int w = 0;
        for (int i = 0; i < o.np; ++i) {
            if (i && lane == 0) alt[w] = ',';
            w += (i ? 1 : 0);
            w += write_piece(S, alt + w, o.q[i]);
        }
    }
    __syncwarp();
    // ---- format_row: filters and genotype
    const uint32_t cfg = p.cfg;
    const bool f_homo_snp = flags >> 1 & 1, f_het_snp = flags >> 2 & 1, f_homo_ins = flags >> 3 & 1, f_het_acgt_ins = flags >> 4 & 1,
               f_het_insins = flags >> 5 & 1, f_homo_del = flags >> 6 & 1, f_het_acgt_del = flags >> 7 & 1,
               f_het_deldel = flags >> 8 & 1, f_insdel = flags >> 9 & 1, f_ref = flags & 1;
    bool multi = false;
    for (int i = lane; i < alt_len; i += 32) multi |= alt[i] == ',';
    multi = __any_sync(0xffffffffu, multi);
    bool same = ref_len == alt_len;
    if (same) {
        bool diff = false;
        for (int i = lane; i < ref_len; i += 32) diff |= ref[i] != alt[i];
        same = !__any_sync(0xffffffffu, diff);
    }
    const bool het = f_het_snp || f_het_acgt_ins || f_het_insins || f_het_acgt_del || f_het_deldel || f_insdel;
    bool printed = !((!(cfg & C3B_CALL_SHOW_REF) && f_ref) || (!f_ref && same));
    if ((cfg & C3B_CALL_HAPLOID_PRECISE) && het) printed = false;
    if ((cfg & C3B_CALL_HAPLOID_SENSITIVE) && multi) printed = false;
    int gt = 255;
    if (f_ref) gt = 0;
    else if (f_homo_snp || f_homo_ins || f_homo_del) gt = 2;
    else if (f_het_snp || f_het_acgt_ins || f_het_insins || f_het_acgt_del || f_het_deldel) gt = 1;
    if (multi) gt = 3;
    int err = printed && (S.bad_empty || S.bad_x) ? 2 : 0;       // format_row reads key[0] and the SNP keys' key[1]
    // ---- format_row: AD and the AF support
    const Rows R{S, (cfg & C3B_CALL_LONG_INDEL) != 0};
    const int ra = warp_best(na, false, [&](int x) { return S.t[x].kind == 'R' ? 0LL : kNone; });
    const long long ref_count = ra < 0 ? 0 : max(0LL, S.t[ra].count);
    long long support = 0;
    int n_ad = 0;
    auto put = [&](long long v) { if (lane == 0) ad[n_ad] = v; ++n_ad; };
    // the pieces of alt.split(",")
    auto for_pieces = [&](auto f) {
        int b = 0;
        for (int i = 0; i <= alt_len; ++i)
            if (i == alt_len || alt[i] == ',') { f(alt + b, i - b); b = i + 1; }
    };
    const long long n_dels = warp_sum(na, [&](int x) { return S.t[x].kind == 'D' ? 1LL : 0LL; });
    if (!printed) {
        // format_row returns before it counts: AD and support stay empty
    } else if (f_ref) {
        support = ref_count;
    } else if (f_homo_snp || f_het_snp) {
        for (int i = 0; i < alt_len; ++i)
            if (alt[i] != ',') { const long long v = R.snp(alt[i]); put(v); support += v; }
    } else if (f_homo_ins || f_het_insins) {
        for_pieces([&](const char *s, int n) { const long long v = R.get('I', s, n) + R.long_ins(s, n); put(v); support += v; });
    } else if (f_het_acgt_ins) {
        const char *s = alt;
        int n = alt_len;
        long long n_snp = 0;
        if (multi) {
            int c = 0;
            while (alt[c] != ',') ++c;
            if (c == 0) err = err ? err : (printed ? 2 : 0);
            else n_snp = R.snp(alt[0]);
            s = alt + c + 1;
            int e = c + 1;
            while (e < alt_len && alt[e] != ',') ++e;
            n = e - (c + 1);
            if (c) put(n_snp);
        }
        const long long n_ins = R.get('I', s, n) + R.long_ins(s, n);
        support = n_ins + n_snp;
        put(n_ins);
    } else if (f_homo_del || f_het_deldel) {
        if (n_dels) {
            if (f_homo_del) {
                if (ref_len <= 1 && R.long_indel) err = err ? err : (printed ? 3 : 0);
                support = ref_len > 1 ? R.get('D', ref + 1, ref_len - 1) : 0;
                put(support);
            } else if (n_dels > 1) {
                for_pieces([&](const char *, int n) { const long long v = R.del_len((long long)ref_len - n); put(v); support += v; });
            }
        }
    } else if (f_het_acgt_del) {
        long long n_snp = 0;
        bool has_snp = false;
        if (multi) {
            int c = 0;
            while (alt[c] != ',') ++c;
            if (c + 1 >= alt_len || alt[c + 1] == ',') err = err ? err : (printed ? 2 : 0);
            else { has_snp = true; n_snp = R.snp(alt[c + 1]); }
        }
        if (ref_len <= 1 && R.long_indel) err = err ? err : (printed ? 3 : 0);
        const long long n_del = ref_len > 1 ? R.get('D', ref + 1, ref_len - 1) : 0;
        support = n_del + n_snp;
        if (has_snp) put(n_snp);
        put(n_del);
    } else if (f_insdel) {
        for_pieces([&](const char *s, int n) {
            const long long alt_l = (long long)ref_len - n;
            long long v;
            if (alt_l < 0) {
                const int m = ref_len > 1 ? n - (ref_len - 1) : n;
                v = R.get('I', s, m) + R.long_ins(s, m);
            } else {
                v = R.del_len(alt_l);
            }
            put(v);
            support += v;
        });
    }
    if (cfg & (C3B_CALL_HAPLOID_PRECISE | C3B_CALL_HAPLOID_SENSITIVE)) {
        if (gt == 255) err = err ? err : (printed ? 3 : 0);       // "1" in None
        else gt = gt == 0 ? 4 : 5;
    }
    __syncwarp();
    // ---- the row's text: '.' for a reference call, IUPAC -> N
    if (f_ref) {
        if (lane == 0) alt[0] = '.';
        alt_len = 1;
    }
    if (!(cfg & C3B_CALL_KEEP_IUPAC)) {
        const bool dot = alt_len == 1 && alt[0] == '.';
        for (int i = lane; i < ref_len + alt_len; i += 32) {
            if (i >= ref_len && dot) continue;
            const char c = text[i], u = (c >= 'a' && c <= 'z') ? c - 32 : c;
            if (!(u == 'A' || u == 'C' || u == 'G' || u == 'T' || u == 'N' || u == ',' || u == '.')) text[i] = 'N';
        }
    }
    __syncwarp();
    if (lane == 0) {
        c3b_call c;
        memset(&c, 0, sizeof(c));
        c.dp = depth;
        c.support = support;
        c.ref_count = ref_count;
        c.prob = prob;
        c.ref_len = ref_len;
        c.alt_len = alt_len;
        c.n_ad = n_ad;
        c.flags = flags;
        c.genotype = (uint8_t)gt;
        c.printed = printed ? 1 : 0;
        c.status = (uint8_t)err;
        *out = c;
    }
}

__global__ void __launch_bounds__(kCallWarps * 32) decode_calls_kernel(const CallsDev p) {
    const int wib = threadIdx.x >> 5;
    int64_t n = p.max_rows;
    if (p.n_sites) n = max((int64_t)0, min((int64_t)*p.n_sites, p.max_rows));
    const int64_t rows = p.is_ref ? max(p.max_rows, p.batch) : n;
    for (int64_t r = (int64_t)blockIdx.x * kCallWarps + wib; r < rows; r += (int64_t)gridDim.x * kCallWarps) {
        if (r < n) {
            const int64_t site = p.sites ? (int64_t)p.sites[r] : r;
            if (site >= 0 && site < p.batch) decode_site(p, site, r);
        }
        if (p.is_ref && r < p.batch && p.is_ref[r]) decode_site(p, r, -1);
    }
}

// ref_base -> gt21 of ref+ref (0 for a base outside the IUPAC table: its record reports status 5)
__global__ void calls_gt21_kernel(const uint8_t *ref_base, int64_t batch, uint8_t *gt21) {
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < batch; b += (int64_t)gridDim.x * blockDim.x) {
        const int c = acgt_of(ref_base[b]);
        gt21[b] = c == 'C' ? 4 : c == 'G' ? 7 : c == 'T' ? 9 : 0;
    }
}

// stable compaction of the unresolved sites, and each re-rank chunk's share of them
__global__ void __launch_bounds__(1024) calls_compact_kernel(const uint8_t *unresolved, int64_t batch, int32_t *rr, int32_t *n_rr,
                                                             int32_t *n_chunk, int n_chunks, int chunk) {
    __shared__ int warp_cnt[32];
    __shared__ int base_s;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) base_s = 0;
    __syncthreads();
    for (int64_t b0 = 0; b0 < batch; b0 += 1024) {
        const int64_t b = b0 + tid;
        const bool u = b < batch && unresolved[b];
        const unsigned bal = __ballot_sync(0xffffffffu, u);
        if (lane == 0) warp_cnt[warp] = __popc(bal);
        __syncthreads();
        int before = 0, total = 0;
        for (int w = 0; w < 32; ++w) {
            const int c = warp_cnt[w];
            if (w < warp) before += c;
            total += c;
        }
        if (u) rr[base_s + before + __popc(bal & ((1u << lane) - 1u))] = (int32_t)b;
        __syncthreads();
        if (tid == 0) base_s += total;
        __syncthreads();
    }
    if (tid == 0) *n_rr = base_s;
    for (int c = tid; c < n_chunks; c += 1024) n_chunk[c] = max(0, min(chunk, base_s - c * chunk));
}

}  // namespace

namespace {

constexpr int64_t kCallsChunk = 4096;      // sites per full re-rank (804 entries each: ~30 MB of ranked rows at 90 outputs)

struct CallsScratch {
    uint8_t *gt21, *is_ref, *unresolved, *cat, *complete, *fcat, *fcomplete;
    float *ref_prob, *maxprob, *prob, *fprob;
    int32_t *nonref, *rr, *count, *argmax, *counters, *fcount;   // counters: n_nonref, n_rr, then each chunk's share
    uint16_t *idx, *tie, *fidx, *ftie;
    double *qual;
    CallAllele *tab;
    int64_t R, chunks;
    // carves the buffers from base (nullptr: only measures); returns the bytes used
    size_t carve(char *base, int64_t batch, int out_dim, int k, int64_t n_alt_bytes) {
        const size_t B = (size_t)batch, E = out_dim == 90 ? 804 : 24, nh = out_dim == 90 ? 4 : 2;
        R = std::min<int64_t>(batch, kCallsChunk);
        chunks = (batch + kCallsChunk - 1) / kCallsChunk;
        size_t o = 0;
        auto take = [&](size_t bytes) { char *q = base ? base + o : nullptr; o += (bytes + 255) / 256 * 256; return q; };
        gt21 = (uint8_t *)take(B); is_ref = (uint8_t *)take(B); unresolved = (uint8_t *)take(B); complete = (uint8_t *)take(B);
        ref_prob = (float *)take(B * 4); nonref = (int32_t *)take(B * 4); rr = (int32_t *)take(B * 4); count = (int32_t *)take(B * 4);
        argmax = (int32_t *)take(B * nh * 4); maxprob = (float *)take(B * nh * 4); qual = (double *)take(B * 8);
        counters = (int32_t *)take(8 + (size_t)chunks * 4);
        cat = (uint8_t *)take(B * k); idx = (uint16_t *)take(B * k * 2); tie = (uint16_t *)take(B * k * 2); prob = (float *)take(B * k * 4);
        fcat = (uint8_t *)take(R * E); fidx = (uint16_t *)take(R * E * 2); ftie = (uint16_t *)take(R * E * 2);
        fprob = (float *)take(R * E * 4); fcount = (int32_t *)take(R * 4); fcomplete = (uint8_t *)take(R);
        tab = (CallAllele *)take(((size_t)n_alt_bytes + B) * sizeof(CallAllele));
        return o;
    }
};

}  // namespace

size_t c3b_calls_scratch_bytes(int64_t batch, int out_dim, int k, int64_t n_alt_bytes) {
    CallsScratch w;
    return w.carve(nullptr, batch, out_dim, k, n_alt_bytes);
}

int c3b_launch_decode_calls(const float *y, const uint8_t *ref_base, int64_t batch, int out_dim, const char *alt_bytes,
                            const int64_t *alt_offsets, int64_t n_alt_bytes, uint32_t cfg, int64_t max_infer_len, int k,
                            c3b_call *calls, char *text, int64_t *ad, void *scratch, cudaStream_t s) {
    if (batch <= 0) return 0;
    const int E = out_dim == 90 ? 804 : 24;
    CallsScratch w;
    w.carve((char *)scratch, batch, out_dim, k, n_alt_bytes);
    const int64_t R = w.R, chunks = w.chunks;
    uint8_t *gt21 = w.gt21, *is_ref = w.is_ref, *unresolved = w.unresolved, *cat = w.cat, *complete = w.complete;
    uint8_t *fcat = w.fcat, *fcomplete = w.fcomplete;
    float *ref_prob = w.ref_prob, *maxprob = w.maxprob, *prob = w.prob, *fprob = w.fprob;
    int32_t *nonref = w.nonref, *rr = w.rr, *count = w.count, *argmax = w.argmax, *counters = w.counters, *fcount = w.fcount;
    uint16_t *idx = w.idx, *tie = w.tie, *fidx = w.fidx, *ftie = w.ftie;
    double *qual = w.qual;
    CallAllele *tab = w.tab;
    const size_t B = (size_t)batch;

    calls_gt21_kernel<<<(unsigned)std::min<int64_t>((batch + 255) / 256, 1024), 256, 0, s>>>(ref_base, batch, gt21);
    C3B_CUDA(cudaGetLastError());
    if (c3b_launch_decode_stage1(y, gt21, batch, out_dim, is_ref, ref_prob, argmax, maxprob, qual, nonref, counters, s)) return 1;
    if (c3b_launch_decode_stage2(y, gt21, batch, out_dim, nonref, counters, batch, k, cat, idx, prob, tie, count, complete, s)) return 1;
    C3B_CUDA(cudaMemsetAsync(unresolved, 0, B, s));
    CallsDev p;
    p.bytes = alt_bytes; p.off = alt_offsets; p.n_bytes = n_alt_bytes; p.ref_base = ref_base; p.batch = batch;
    p.add_indel = out_dim == 90; p.cfg = cfg; p.max_len = max_infer_len;
    p.is_ref = is_ref; p.ref_prob = ref_prob; p.sites = nonref; p.n_sites = counters; p.max_rows = batch; p.k = k;
    p.cat = cat; p.idx = idx; p.prob = prob; p.tie = tie; p.count = count;
    p.tab = tab; p.unresolved = unresolved; p.calls = calls; p.text = text; p.ad = (long long *)ad;
    const unsigned blocks = (unsigned)std::min<int64_t>((batch + kCallWarps - 1) / kCallWarps, 8192);
    decode_calls_kernel<<<blocks, kCallWarps * 32, 0, s>>>(p);
    C3B_CUDA(cudaGetLastError());
    calls_compact_kernel<<<1, 1024, 0, s>>>(unresolved, batch, rr, counters + 1, counters + 2, (int)chunks, (int)R);
    C3B_CUDA(cudaGetLastError());
    // re-rank: the unresolved sites in chunks of at most R, each ranked in full and walked again
    for (int64_t ch = 0; ch < chunks; ++ch) {
        if (c3b_launch_decode_stage2(y, gt21, batch, out_dim, rr + ch * R, counters + 2 + ch, R, E, fcat, fidx, fprob, ftie,
                                     fcount, fcomplete, s))
            return 1;
        CallsDev q = p;
        q.is_ref = nullptr; q.sites = rr + ch * R; q.n_sites = counters + 2 + ch; q.max_rows = R; q.k = E;
        q.cat = fcat; q.idx = fidx; q.prob = fprob; q.tie = ftie; q.count = fcount;
        decode_calls_kernel<<<(unsigned)std::min<int64_t>((R + kCallWarps - 1) / kCallWarps, 8192), kCallWarps * 32, 0, s>>>(q);
        C3B_CUDA(cudaGetLastError());
    }
    return 0;
}
