// plp_alt_text.cu - the pileup counter's all_alt_info text on the GPU (include/clair3_b200_pileup.h: c3b_plp_alt_text).
//
// Reference: the text loop of calculate_clair3_pileup(), HKU-BAL/Clair3 src/clair3_pileup.c:391-450, one string per candidate:
//     "<pos+1>-<depth>-<REF>-X<b> n D<ref bases> n I<REF><inserted bases> n R<REF> n "
// clair3_b200/pileup_counts.py: format_alt_info / khash_iteration_order state the same on the host and are what the tests hold
// these kernels to.  The stage is alt_text.cuh's measure -> scan -> write (T2 the scans, T3 text_write_kernel); what is the
// pileup counter's own is
//
//   T1 plp_text_measure   one WARP per candidate over the column's allele records (K3's export, [al_off, al_off + al_n)):
//                         lanes over records merge the two strands (a record's twin on the other strand: same kind, length and,
//                         for insertions, the same bases through the representative reads' packed sequences), hash the merged
//                         insertion strings (X31) and rank-sort the deletions by length and the insertions by first read; lane 0
//                         then replays klib's khash (src/khash.h) over the insertions - power-of-two tables from 4, triangular
//                         probing, growth at 0.77 load at the start of a put, kh_resize's in-place kick-out rehash, one more
//                         growth when a put of a present string follows the last new one - and leaves the bucket order.
//   PlpText::emit         the string, from the merged and ordered records.
//
// Everything a column needs lives in global scratch addressed by its own record range (mate / hash / order) or by that range and
// its candidate index (the khash table: 8 buckets per candidate, or up to 3 per record - a table of n > 8 buckets holds at least
// 0.77 n / 2 strings), so a column of thousands of distinct alleles needs no capacity of its own.  The grids are sized from the
// region's width and read n_cand on the device.
#include "alt_text.cuh"

namespace {

constexpr int FETCH_EXPAND = 1000;                        // mpileup_expand_reference_region, src/clair3_pileup.h:63
constexpr int32_t NOT_FIRST = -2;                         // mate[]: the record's twin comes earlier in the list

__device__ __forceinline__ int64_t first_read(const PlpAltTextArgs &A, int i) {
    const int m = A.mate[i];
    const uint32_t r = A.al_read[i];
    return (int64_t)(m >= 0 && A.al_read[m] < r ? A.al_read[m] : r);
}
__device__ __forceinline__ long long merged_count(const PlpAltTextArgs &A, int i) {
    const int m = A.mate[i];
    return (long long)A.al_cnt[i] + (m >= 0 ? (long long)A.al_cnt[m] : 0);
}

// The stage for alt_text.cuh: the candidate count is the count's device counter.
struct PlpText {
    typedef PlpAltTextArgs Args;
    static __device__ __forceinline__ int64_t n_cand(const Args &A) { return *A.n_cand; }
    static const int64_t *n_cand_dev(const Args &A) { return A.n_cand; }
    static __device__ __forceinline__ int64_t pos(const Args &A, int64_t j) { return A.major[A.cand_cols[j]]; }
    // upper_base of the reference base under a column, 'N' outside the supplied reference
    static __device__ __forceinline__ int ref_base(const Args &A, int64_t pos) {
        const int64_t off = pos - A.ref_start;
        const int rb = (off >= 0 && off < A.ref_len) ? (int)(unsigned char)A.ref[off] : 'N';
        return rb >= 'a' && rb <= 'z' ? rb - 32 : rb;
    }
    template <class S> static __device__ void emit(const Args &A, int64_t j, int ni, int nd, TextOut<S> &o);
};

// One candidate's string, src/clair3_pileup.c:391-450, from the merged and ordered allele records T1 left in `order`: ni
// insertions in bucket order, then nd deletions by length.
template <class S> __device__ void PlpText::emit(const Args &A, const int64_t j, const int ni, const int nd, TextOut<S> &o) {
    const int64_t ci = A.cand_cols[j], pos = A.major[ci], off = pos - A.ref_start;
    const int a0 = A.al_off[pos - A.start];
    const int rb = ref_base(A, pos);
    const int bi = rb - 'A';
    const int rf = bi == 2 ? 1 : bi == 6 ? 2 : bi == 19 ? 3 : 0;          // base2index, src/clair3_pileup.h:57-62
    const long long depth = A.stats[ci * 6];
    long long ref_depth = A.stats[ci * 6 + 1];
    typedef TextOut<S> O;
    o.num(pos + 1, O::HEAD_FULL); o.head('-', false);                     // "<pos+1>-<depth>-<REF>-" / "<depth>-"
    o.num(depth, O::HEAD_BOTH); o.head('-', true);
    o.head((char)rb, false); o.head('-', false);
    const int64_t *row = A.matrix + ci * 18;
    for (int i = 0; i < 4; ++i) {
        const long long alt_sum = (long long)row[i] + (long long)row[i + 9];
        if (alt_sum > 0 && i != rf) {
            o.alt('X'); o.alt("ACGT"[i]); o.alt(' '); o.num(alt_sum, O::ALT); o.alt(' ');
        }
    }
    for (int k = 0; k < nd; ++k) {                                        // deletions, ascending length
        const int i = A.order[a0 + ni + k];
        const long long len = (long long)(A.al_meta[i] & 0x3fffffffu), d = merged_count(A, i);
        ref_depth -= d;
        if (d > 0 && len <= A.max_indel_length) {
            int64_t stop = off + 1 + len;                                 // the reference's FASTA fetch ends at end + 1000
            if (stop > A.end + FETCH_EXPAND + 1 - A.ref_start) stop = A.end + FETCH_EXPAND + 1 - A.ref_start;
            if (stop > A.ref_len) stop = A.ref_len;
            o.alt('D');
            for (int64_t q = off + 1; q < stop; ++q) {
                const char c = A.ref[q];
                if (c == 0) break;
                o.alt(c);
            }
            o.alt(' '); o.num(d, O::ALT); o.alt(' ');
        }
    }
    for (int k = 0; k < ni; ++k) {                                        // insertions, khash bucket order
        const int i = A.order[a0 + k];
        const long long len = (long long)(A.al_meta[i] & 0x3fffffffu), v = merged_count(A, i);
        ref_depth -= v;
        if (len <= A.max_indel_length) {
            const uint32_t r = A.al_read[i];
            const uint8_t *sq = A.R.seq + A.R.seq_off[r];
            const int lq = A.R.l_qseq[r];
            const long long q0 = (long long)A.al_qpos[i];
            o.alt('I'); o.alt((char)rb);
            for (long long q = 0; q < len; ++q) o.alt(NT16[c3b_nib_at(sq, lq, q0 + q)]);
            o.alt(' '); o.num(v, O::ALT); o.alt(' ');
        }
    }
    if (ref_depth > 0) {
        o.alt('R'); o.alt((char)rb); o.alt(' '); o.num(ref_depth, O::ALT); o.alt(' ');
    }
}

// ---------------------------------------------------------------------------------------------------------------- T1
__global__ void __launch_bounds__(256) plp_text_measure_kernel(PlpAltTextArgs A) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int64_t n_cand = *A.n_cand;
    for (int64_t j = warp; j <= n_cand; j += nwarps) {
        if (j == n_cand) {                                    // the scans run over n_cand + 1 entries: the last offset is the total
            if (lane == 0) A.len_text[j] = A.len_dec[j] = 0;
            continue;
        }
        const int64_t ci = A.cand_cols[j], pos = A.major[ci];
        const int a0 = A.al_off[pos - A.start];
        int n = A.al_n[pos - A.start];
        bool fits = (int64_t)a0 + n <= A.al_cap;              // mate / hash / order / table hold al_cap records
        if (!fits) n = 0;
        // a record's twin on the other strand (K3 keeps each strand's alleles distinct, so there is at most one)
        int ni = 0, nd = 0;
        for (int i = a0 + lane; i < a0 + n; i += 32) {
            const uint32_t meta = A.al_meta[i];
            const long long len = (long long)(meta & 0x3fffffffu);
            const bool ins = meta >> 31;
            const uint8_t *sq = nullptr;
            int lq = 0;
            long long q0 = 0;
            if (ins) {
                sq = A.R.seq + A.R.seq_off[A.al_read[i]];
                lq = A.R.l_qseq[A.al_read[i]];
                q0 = (long long)A.al_qpos[i];
            }
            int m = -1;
            for (int k = a0; k < a0 + n && m == -1; ++k) {
                if (A.al_meta[k] != (meta ^ (1u << 30))) continue;
                bool same = true;
                if (ins) {
                    const uint8_t *s2 = A.R.seq + A.R.seq_off[A.al_read[k]];
                    const int lq2 = A.R.l_qseq[A.al_read[k]];
                    const long long q2 = (long long)A.al_qpos[k];
                    for (long long q = 0; q < len; ++q)
                        if (c3b_nib_at(sq, lq, q0 + q) != c3b_nib_at(s2, lq2, q2 + q)) { same = false; break; }
                }
                if (same) m = k < i ? NOT_FIRST : k;
            }
            A.mate[i] = m;
            if (m != NOT_FIRST) {
                if (ins) {                                    // __ac_X31_hash_string, src/khash.h:395-400
                    uint32_t h = len ? (uint32_t)NT16[c3b_nib_at(sq, lq, q0)] : 0u;
                    for (long long q = 1; q < len; ++q) h = h * 31u + (uint32_t)NT16[c3b_nib_at(sq, lq, q0 + q)];
                    A.hash[i] = h;
                    ++ni;
                } else {
                    ++nd;
                }
            }
        }
#pragma unroll
        for (int d = 16; d; d >>= 1) {
            ni += __shfl_xor_sync(0xffffffffu, ni, d);
            nd += __shfl_xor_sync(0xffffffffu, nd, d);
        }
        __syncwarp();
        // rank sort: deletions by length, insertions by first occurrence over both strands (the reference's insertion order)
        for (int i = a0 + lane; i < a0 + n; i += 32) {
            if (A.mate[i] == NOT_FIRST) continue;
            const uint32_t meta = A.al_meta[i];
            const bool ins = meta >> 31;
            const int64_t key = ins ? first_read(A, i) : (int64_t)(meta & 0x3fffffffu);
            int rank = 0;
            for (int k = a0; k < a0 + n; ++k) {
                if (A.mate[k] == NOT_FIRST || (A.al_meta[k] >> 31) != (meta >> 31)) continue;
                const int64_t kk = ins ? first_read(A, k) : (int64_t)(A.al_meta[k] & 0x3fffffffu);
                rank += (kk < key || (kk == key && k < i)) ? 1 : 0;
            }
            A.order[a0 + (ins ? 0 : ni) + rank] = i;
        }
        __syncwarp();
        if (lane == 0) {
            if (ni > 0 && fits) {                             // the khash replay: a short serial walk
                uint32_t *slot = A.table + 8 * j;
                int avail = 8;
                if (ni > 3) { slot = A.table + 8 * A.n + 3 * (int64_t)a0; avail = 3 * n; }
                // a read after the last new string put a present one again: that put still grows a full table first
                const bool again = (int64_t)A.ins_last[pos - A.start] > first_read(A, A.order[a0 + ni - 1]);
                fits = khash_replay(A.hash, A.order + a0, ni, again, slot, avail);
            }
            text_measure_tail<PlpText>(A, j, fits, ni, nd);
        }
    }
}

}  // namespace

int c3b_launch_plp_alt_text(const PlpAltTextArgs &a, cudaStream_t s, int *launches) {
    return text_launch<PlpText>(a, plp_text_measure_kernel, s, launches, "c3b_plp_alt_text");
}
