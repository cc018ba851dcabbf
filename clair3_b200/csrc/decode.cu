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
