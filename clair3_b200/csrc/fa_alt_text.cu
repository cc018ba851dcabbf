// fa_alt_text.cu - the full-alignment builder's all_alt_info text on the GPU (include/clair3_b200_fa.h: c3b_fa_alt_text).
//
// Reference: the text loop of calculate_clair3_full_alignment(), HKU-BAL/Clair3 src/clair3_full_alignment_dwell.c:950-1006, one
// string per candidate:
//     "<cand+1>-<depth>-<REF>-X<b> n I<REF><inserted bases> n D<ref bases> n R<REF> n "
// clair3_b200/fa_tensor.py: format_alt_info / khash_iteration_order state the same on the host and are what the tests hold these
// kernels to.  K11 (fa_candidate_kernel) already exports each candidate's depth, A/C/G/T counts and its distinct indel alleles,
// merged over the strands and in put order (the order in which the reference's two khash counters saw them).  The stage is
// alt_text.cuh's measure -> scan -> write (F2 the scans, F3 text_write_kernel); what is the builder's own is
//
//   F1 fa_text_measure    one WARP per candidate over its allele records [al_off, al_off + al_n): lanes hash them (X31 over the
//                         NT16 bases of an insertion string, the length of a deletion: kh_int_hash_func) and split them, in put
//                         order, into the insertions and then the deletions; lane 0 replays the two khash tables (alt_text.cuh).
//   FaText::emit          the string, from the candidate's counters and its ordered records.
//
// Scratch is global and addressed by the candidate's own record range (hash / order) or by that range and the candidate index
// (the khash table: 8 buckets per candidate, or up to 3 per record; both tables of a candidate use the same buckets, one after
// the other), so a candidate with thousands of distinct alleles needs no capacity of its own.  The candidate count is a host value.
#include "alt_text.cuh"

namespace {

// The stage for alt_text.cuh: the candidate count is known on the host.
struct FaText {
    typedef FaAltTextArgs Args;
    static __device__ __forceinline__ int64_t n_cand(const Args &A) { return A.n; }
    static const int64_t *n_cand_dev(const Args &) { return nullptr; }
    static __device__ __forceinline__ int64_t pos(const Args &A, int64_t j) { return A.cand[j]; }
    // upper_base of the reference base under a candidate, '\0' outside the supplied reference (as the host formatter writes it)
    static __device__ __forceinline__ char ref_base(const Args &A, int64_t pos) {
        const int64_t off = pos - A.ref_start;
        const char c = (off >= 0 && off < A.ref_len) ? A.ref[off] : '\0';
        return (c >= 'a' && c <= 'z') ? (char)(c - 32) : c;
    }
    template <class S> static __device__ void emit(const Args &A, int64_t j, int ni, int nd, TextOut<S> &o);
};

// One candidate's string, src/clair3_full_alignment_dwell.c:950-1006, from its counters and the allele records F1 left in
// `order`: ni insertions, then nd deletions, each kind in bucket order.
template <class S> __device__ void FaText::emit(const Args &A, const int64_t j, const int ni, const int nd, TextOut<S> &o) {
    const int64_t c = A.cand[j], off = c - A.ref_start;
    const int a0 = A.al_off[j];
    const char rb = ref_base(A, c);
    const int rf = rb == 'C' ? 1 : rb == 'G' ? 2 : rb == 'T' ? 3 : 0;    // acgt2num, src/clair3_full_alignment_dwell.h:49-54
    const int32_t *acgt = A.c_acgt + 4 * j;
    long long ref_count = acgt[rf];
    typedef TextOut<S> O;
    o.num(c + 1, O::HEAD_FULL); o.head('-', false);                       // "<cand+1>-<depth>-<REF>-" / "<depth>-"
    o.num(A.c_depth[j], O::HEAD_BOTH); o.head('-', true);
    o.head(rb, false); o.head('-', false);
    if (rb == '-') o.cut = true;             // split("-") then reads the REF field and the alt field as empty strings
    for (int i = 0; i < 4; ++i) {
        if (i != rf && acgt[i] > 0) {
            o.alt('X'); o.alt("ACGT"[i]); o.alt(' '); o.num(acgt[i], O::ALT); o.alt(' ');
        }
    }
    for (int k = 0; k < ni; ++k) {                                        // insertions, bucket order of the string counter
        const int i = A.order[a0 + k];
        const long long len = (long long)(A.al_meta[i] & 0x3fffffffu), v = A.al_cnt[i];
        ref_count -= v;
        if (len <= A.max_indel_length) {
            const uint32_t r = A.al_read[i];
            const uint8_t *sq = A.R.seq + A.R.seq_off[r];
            const int lq = A.R.l_qseq[r];
            const long long q0 = (long long)A.al_qpos[i];
            o.alt('I'); o.alt(rb);
            for (long long q = 0; q < len; ++q) o.alt(NT16[c3b_nib_at(sq, lq, q0 + q)]);
            o.alt(' '); o.num(v, O::ALT); o.alt(' ');
        }
    }
    for (int k = 0; k < nd; ++k) {                                        // deletions, bucket order of the int counter
        const int i = A.order[a0 + ni + k];
        const long long len = (long long)(A.al_meta[i] & 0x3fffffffu), v = A.al_cnt[i];
        ref_count -= v;
        if (len <= A.max_indel_length) {
            // "D%.*s": up to len bases after the candidate, to the end of the supplied reference or its first NUL
            int64_t q = off + 1 < 0 ? 0 : off + 1;
            const int64_t stop = off + 1 + len < A.ref_len ? off + 1 + len : A.ref_len;
            o.alt('D');
            for (; q < stop; ++q) {
                const char ch = A.ref[q];
                if (ch == 0) break;
                o.alt(ch);
            }
            o.alt(' '); o.num(v, O::ALT); o.alt(' ');
        }
    }
    if (ref_count > 0) {
        o.alt('R'); o.alt(rb); o.alt(' '); o.num(ref_count, O::ALT); o.alt(' ');
    }
}

// ---------------------------------------------------------------------------------------------------------------- F1
__global__ void __launch_bounds__(256) fa_text_measure_kernel(FaAltTextArgs A) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t j = warp; j <= A.n; j += nwarps) {
        if (j == A.n) {                                       // the scans run over n_cand + 1 entries: the last offset is the total
            if (lane == 0) A.len_text[j] = A.len_dec[j] = 0;
            continue;
        }
        const int a0 = A.al_off[j];
        int n = A.al_n[j];
        bool fits = (int64_t)a0 + n <= A.al_cap;              // hash / order / table hold al_cap records
        if (!fits) n = 0;
        // hashes (kh_str_hash_func = __ac_X31_hash_string, src/khash.h:395-400; kh_int_hash_func: the key), and which kind
        // saw a put of a present key after its last new one (bit 30 of that kind's last record)
        int ni = 0;
        bool again_i = false, again_d = false;
        for (int i = a0 + lane; i < a0 + n; i += 32) {
            const uint32_t meta = A.al_meta[i];
            const uint32_t len = meta & 0x3fffffffu;
            uint32_t h = len;
            if (meta >> 31) {
                const uint32_t r = A.al_read[i];
                const uint8_t *sq = A.R.seq + A.R.seq_off[r];
                const int lq = A.R.l_qseq[r];
                const long long q0 = (long long)A.al_qpos[i];
                h = len ? (uint32_t)NT16[c3b_nib_at(sq, lq, q0)] : 0u;
                for (long long q = 1; q < (long long)len; ++q) h = h * 31u + (uint32_t)NT16[c3b_nib_at(sq, lq, q0 + q)];
                ++ni;
                again_i |= (meta >> 30) & 1u;
            } else {
                again_d |= (meta >> 30) & 1u;
            }
            A.hash[i] = h;
        }
#pragma unroll
        for (int d = 16; d; d >>= 1) ni += __shfl_xor_sync(0xffffffffu, ni, d);
        again_i = __any_sync(0xffffffffu, again_i);
        again_d = __any_sync(0xffffffffu, again_d);
        // put order within each kind: the insertions to order[a0, a0 + ni), the deletions after them
        int base_i = a0, base_d = a0 + ni;
        for (int i0 = a0; i0 < a0 + n; i0 += 32) {
            const int i = i0 + lane;
            const bool in = i < a0 + n;
            const bool ins = in && (A.al_meta[i] >> 31);
            const unsigned mi = __ballot_sync(0xffffffffu, ins), md = __ballot_sync(0xffffffffu, in && !ins);
            const unsigned below = (1u << lane) - 1u;
            if (ins) A.order[base_i + __popc(mi & below)] = i;
            else if (in) A.order[base_d + __popc(md & below)] = i;
            base_i += __popc(mi);
            base_d += __popc(md);
        }
        __syncwarp();
        if (lane == 0) {
            const int nd = n - ni;
            if (fits && n > 0) {                              // the two khash replays: short serial walks on the same buckets
                uint32_t *slot = A.table + 8 * j;
                int avail = 8;
                if (ni > 3 || nd > 3) { slot = A.table + 8 * A.n + 3 * (int64_t)a0; avail = 3 * n; }
                fits = khash_replay(A.hash, A.order + a0, ni, again_i, slot, avail) &&
                       khash_replay(A.hash, A.order + a0 + ni, nd, again_d, slot, avail);
            }
            text_measure_tail<FaText>(A, j, fits, ni, nd);
        }
    }
}

}  // namespace

int c3b_launch_fa_alt_text(const FaAltTextArgs &a, cudaStream_t s, int *launches) {
    return text_launch<FaText>(a, fa_text_measure_kernel, s, launches, "c3b_fa_alt_text");
}
