// Internal declarations shared by the C-ABI translation unit and the kernel files.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <map>
#include <string>
#include <vector>

#include "../../include/clair3_b200.h"
#include "../../include/clair3_b200_debug.h"
#include "../../include/clair3_b200_fa.h"
#include "../../include/clair3_b200_pileup.h"
#include "records_check.cuh"

#define C3B_T 33            // positions per site (shared/param_p.py:34-35)
#define C3B_H1 128          // LSTM1 hidden (clair3/model.py:46)
#define C3B_H2 160          // LSTM2 hidden (clair3/model.py:47)
#define C3B_MAX_HEADS 4
#define C3B_X1_COLS 48      // LSTM1 x operand columns: [hi(x) (channels) | 1 | lo(x) (channels) | 0...]  (lstm_tc.cu)
#define C3B_MAX_PILEUP_CHANNELS ((C3B_X1_COLS - 1) / 2)

void c3b_set_error(const char *fmt, ...);
void c3b_note_grid(long long ctas);      // launchers report their grid size (CTAs) for the per-kernel profile (SM-time = CTAs x duration)

// Tensor-core operand type.  fp16 (11-bit significand) rather than bf16 (8-bit): same wgmma rate, 8x smaller rounding
// error; every operand on this path is bounded (counts <= 2048 exact, |h| <= 1, BN-normalised feature maps) and stores
// saturate at +-65504 instead of overflowing.
typedef __half op_t;
typedef __half2 op2_t;
#ifdef __CUDACC__
__device__ __forceinline__ float op_clamp(float x) { return fminf(fmaxf(x, -65504.f), 65504.f); }
__device__ __forceinline__ op_t f2op(float x) { return __float2half_rn(x); }
// saturating variant for values that are not bounded by construction (raw input counts): +-65504 instead of inf
__device__ __forceinline__ op_t f2op_sat(float x) {
    unsigned short r;
    asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(r) : "f"(x));
    return __ushort_as_half(r);
}
__device__ __forceinline__ op2_t f2op2(float a, float b) { return __floats2half2_rn(a, b); }
__device__ __forceinline__ float2 op22f2(op2_t v) { return __half22float2(v); }
// two floats -> packed fp16 pair in ONE instruction, saturating at +-65504 instead of overflowing to inf
__device__ __forceinline__ uint32_t f2op2_sat(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}
__device__ __forceinline__ float op2f(op_t v) { return __half2float(v); }
#endif
// "Tile-major k-group-planar" activation matrices (h1, h2, spp): [row tile of 128][K/8 k-groups][128 rows][8] fp16.  A GEMM
// tile's 64-wide k-chunk (8 k-groups) is then ONE contiguous 16 KB run = one cp.async.bulk instead of eight 2 KB ones.
// Returns the element offset of (row, k-group kg, lane 0).
#ifdef __CUDACC__
__host__ __device__
#endif
inline size_t c3b_tile_major_offset(size_t row, int kg, int kgroups) {
    return (((row >> 7) * (size_t)kgroups + (size_t)kg) * 128 + (row & 127)) * 8;
}
uint16_t c3b_f2op(float f);     // host: fp32 -> fp16 bits, round-to-nearest-even, saturating
// Torch gate row (gate*H + unit) of row R in [0, 4H) of the recurrent kernels' permuted gate order (lstm_tc.cu): 64-row block
// 2p holds gates i (rows 16w + q, q < 8) and f (rows 16w + q + 8) of units 32p + 8w + q, block 2p + 1 gates g and o.
inline int c3b_lstm_row(int R, int H) {
    const int pp = R / 128, blk = (R / 64) & 1, r = R % 64, w = r / 16, q = r % 16;
    return (2 * blk + (q >= 8)) * H + 32 * pp + 8 * w + (q & 7);
}
// Torch gate row of LSTM2 pre-gate column C in [0, 640) of one direction (the output columns of proj2): "gate-quad" order, the
// four gates i, f, g, o of unit 32p + u (u < 32) in the adjacent columns 128p + 4u .. +3, so the recurrent kernel's thread that
// owns the unit in block pair p reads them with one 8-byte load.
inline int c3b_lstm2_pg_row(int C) {
    return (C & 3) * C3B_H2 + 32 * (C >> 7) + ((C & 127) >> 2);
}
float c3b_op2f(uint16_t h);     // host: fp16 bits -> fp32

#define C3B_CUDA(expr)                                                                          \
    do {                                                                                        \
        cudaError_t _e = (expr);                                                                \
        if (_e != cudaSuccess) {                                                                \
            c3b_set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return 1;                                                                           \
        }                                                                                       \
    } while (0)

// A device buffer that grows on demand and frees itself.  Sizing::exact grows to the size asked for: the model's weights,
// workspace and staging, whose sizes follow the call shape, which rarely changes.  Sizing::headroom adds 25 %: the pileup
// counter's and the full-alignment builder's per-call buffers, whose sizes follow the data of each call.  Growing first waits
// for stream s, on which queued work may still use the old memory.  `what` names the owner in the error message.
struct C3bBuf {
    enum Sizing { headroom, exact };
    const Sizing sizing;
    void *p = nullptr;
    size_t cap = 0;
    explicit C3bBuf(Sizing z = headroom) : sizing(z) {}
    C3bBuf(const C3bBuf &) = delete;
    C3bBuf &operator=(const C3bBuf &) = delete;
    ~C3bBuf() { if (p) cudaFree(p); }
    int ensure(size_t bytes, cudaStream_t s, const char *what) {
        if (bytes <= cap) return 0;
        if (p) {
            C3B_CUDA(cudaStreamSynchronize(s));
            cudaFree(p);
        }
        p = nullptr;
        cap = 0;
        const size_t want = sizing == exact ? bytes : bytes + bytes / 4 + 256;
        if (cudaMalloc(&p, want) != cudaSuccess) {
            c3b_set_error("%s: cudaMalloc of %zu bytes failed", what, want);
            return 1;
        }
        cap = want;
        return 0;
    }
    template <class T> T *as() const { return reinterpret_cast<T *>(p); }
};

// One input array of a call: a device pointer passes through, host memory is copied into b on stream s.
template <class T>
int c3b_upload(C3bBuf &b, const T *src, size_t bytes, int on_device, const T *&dev, cudaStream_t s, const char *what) {
    if (on_device) { dev = src; return 0; }
    if (b.ensure(bytes ? bytes : 1, s, what)) return 1;
    if (bytes) C3B_CUDA(cudaMemcpyAsync(b.p, src, bytes, cudaMemcpyHostToDevice, s));
    dev = b.as<const T>();
    return 0;
}

// The alignment records as the pileup counter's and the full-alignment builder's kernels read them: the c3b_bam_records arrays
// and c3b_fa_records' optional fields, all device pointers; an optional field is null when the call has none.
struct C3bReads {
    int64_t n;
    const int64_t *pos;
    const uint16_t *flag;
    const uint8_t *mapq;
    const int64_t *cigar_off;
    const uint32_t *cigar;
    const int64_t *seq_off;
    const uint8_t *seq;
    const int32_t *l_qseq;
    const int64_t *qual_off;
    const uint8_t *qual;
    const int64_t *qname_off;
    const uint8_t *qname;
    const int64_t *mv_off;
    const int32_t *mv;
};

#ifdef __CUDACC__
// 4-bit nt16 code of base i of a packed sequence (bam_get_seq: two per byte, high nibble first) of lq bases; 0 ('=') outside it
__device__ __forceinline__ int c3b_nib_at(const uint8_t *sq, int lq, long long i) {
    if (i < 0 || i >= lq) return 0;
    return (__ldg(sq + (i >> 1)) >> ((~i & 1) << 2)) & 15;
}
#endif

// The fault key (records_check.cuh) of records on the device: runs records_check_kernel on stream s into the 8 bytes of
// `scratch` and waits for it.  Launches nothing for a run with nothing to check.
int c3b_records_check_device(const C3bRecordsView &v, C3bBuf &scratch, cudaStream_t s, uint64_t *key);

// Makes device `ordinal` current after checking that it exists and is an sm_90 part.  Returns 0; `unsupported` when there
// is no CUDA device or it is not sm_90; 1 for a bad ordinal or a failed runtime call.  sm_count (optional): its SM count.
int c3b_use_device(int ordinal, int unsupported, int *sm_count);

constexpr int C3B_AL_CAP = 1 << 22;     // allele records the pileup counter or the full-alignment builder exports per call

// What both all_alt_info text stages (alt_text.cuh) take: the records and the reference where the count or build left them, the
// exported allele records, the stage's scratch and outputs, and its status word and byte totals in the counter block.  The
// pileup counter's PlpAltTextArgs and the full-alignment builder's FaAltTextArgs add their own candidate data.
struct C3bAltText {
    int64_t n;                          // the bound on the candidates the grids and buffers are sized from
    int64_t ref_start, ref_len, max_indel_length;
    const char *ref;
    C3bReads R;
    const int32_t *al_off, *al_n;       // per column / candidate: its first record and number of records
    const uint32_t *al_meta, *al_read, *al_qpos, *al_cnt;
    int64_t al_cap;                     // records the al_* arrays and the per-record scratch hold
    // scratch
    uint32_t *hash;                     // [al_cap]
    int32_t *order;                     // [al_cap]
    uint32_t *table;                    // [8 * n + 3 * al_cap] khash buckets
    int32_t *n_ins, *n_del;             // [n]
    int32_t *len_text, *len_dec;        // [n + 1]
    int *status;                        // the stage's status word: non-zero = a candidate's text did not fit the stage's buffers
    // outputs
    char *text, *dec;
    int64_t text_cap, dec_cap;
    int64_t *text_off, *dec_off;        // [n + 1]
    int64_t *totals;                    // device: n_text_bytes, n_decoder_bytes
    uint8_t *ref_base;                  // [n]
    int64_t *position;                  // [n]
};

// What the pileup counter (c3b_plp) and the full-alignment builder (c3b_fa) hold alike: the device and the stream of the last
// call, a pair of CUDA events around each timed stage with the stage's kernel launches, a device counter block with its pinned
// host mirror, the record intake, the exported allele records, and the all_alt_info text stage (stage 1).  The destructor
// releases the events and the pinned memory.  The BAM reader (c3b_bam) uses the events and the counter block; its intake buffers
// stay unallocated.
struct C3bRegionWorkspace {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[2][2] = {};           // per stage: start, end
    int launches[2] = {};
    C3bBuf counters;
    int64_t *host_counters = nullptr;    // pinned copy of `counters`
    int n_counters = 0;
    int text_word = 0;                   // counters[text_word .. +2]: the text stage's status, text bytes, decoder bytes
    C3bBuf al_meta, al_read, al_qpos, al_cnt, al_off, al_n;
    // the records and the reference of the last count / build where they live on the device (intake), with the CIGAR words and
    // sequence bytes the records hold, and the device copies of the host arrays among them
    C3bReads R{};
    const char *dref = nullptr;
    int64_t ref_start = 0, ref_len = 0, n_cigar = 0, n_seq = 0;
    C3bBuf in_core[8], in_qoff, in_qual, in_noff, in_name, in_moff, in_mv, in_ref, in_check;
    // the text stage's scratch and outputs
    C3bBuf tx_hash, tx_order, tx_table, tx_nins, tx_ndel, tx_len_text, tx_len_dec;
    C3bBuf tx_text, tx_dec, tx_text_off, tx_dec_off, tx_ref_base, tx_position;
    bool texted = false;

    C3bRegionWorkspace() = default;
    C3bRegionWorkspace(const C3bRegionWorkspace &) = delete;
    C3bRegionWorkspace &operator=(const C3bRegionWorkspace &) = delete;
    ~C3bRegionWorkspace() {
        for (auto &p : ev)
            for (cudaEvent_t e : p)
                if (e) cudaEventDestroy(e);
        if (host_counters) cudaFreeHost(host_counters);
    }
    // Device time between the events of stage i, after waiting for its end, and the stage's launches.
    int elapsed(int i, float *ms, int *n) {
        C3B_CUDA(cudaSetDevice(device));
        C3B_CUDA(cudaEventSynchronize(ev[i][1]));
        float t = 0.f;
        C3B_CUDA(cudaEventElapsedTime(&t, ev[i][0], ev[i][1]));
        if (ms) *ms = t;
        if (n) *n = launches[i];
        return 0;
    }
    // Queues the copy of the first `bytes` of src into dst on the workspace's stream; nothing for a null dst or no bytes.
    int get(void *dst, const C3bBuf &src, size_t bytes) {
        if (dst && bytes) C3B_CUDA(cudaMemcpyAsync(dst, src.p, bytes, cudaMemcpyDeviceToHost, stream));
        return 0;
    }
    int wait() {
        C3B_CUDA(cudaStreamSynchronize(stream));
        return 0;
    }
    // Queues the copies of the first n allele records into whichever of meta / read / qpos / cnt is given; `who` names the
    // entry point in the error when they hold fewer than n.
    int get_alleles(const char *who, int64_t n, int64_t capacity, uint32_t *meta, uint32_t *read, uint32_t *qpos, uint32_t *cnt) {
        if (!meta && !read && !qpos && !cnt) return 0;
        if (capacity < n) { c3b_set_error("%s: capacity %lld < %lld records", who, (long long)capacity, (long long)n); return 1; }
        const size_t b = (size_t)n * 4;
        return get(meta, al_meta, b) || get(read, al_read, b) || get(qpos, al_qpos, b) || get(cnt, al_cnt, b);
    }

    // The records and the reference of a count / build on `stream`: checks the records (n_reads below max_reads, no null array
    // when there are reads, then everything records_check.cuh checks: on the host for host records, for device records in one
    // kernel whose verdict the call waits for) and the reference, copies host arrays to the device in field order, the
    // reference last, and fills R, dref, ref_start, ref_len, n_cigar and n_seq.  Nothing is copied or launched after a failed
    // check.  opt: the optional fields, null for none; mv only with want_mv.  `who` names the entry point in the errors.
    int intake(const char *who, const c3b_bam_records *core, const c3b_fa_records *opt, bool want_mv, int64_t max_reads,
               int on_device, const char *ref_seq, int64_t ref_start, int64_t ref_len) {
        const int64_t n = core->n_reads;
        if (n < 0 || n >= max_reads) { c3b_set_error("%s: bad n_reads", who); return 1; }
        if (n > 0 && (!core->pos || !core->flag || !core->mapq || !core->cigar_off || !core->cigar || !core->seq_off ||
                      !core->seq || !core->l_qseq)) {
            c3b_set_error("%s: null record array", who);
            return 1;
        }
        if (ref_len > 0 && !ref_seq) { c3b_set_error("%s: null ref_seq", who); return 1; }
        uint64_t fault = C3B_REC_OK;
        if (!on_device) fault = c3b_records_check(core, opt);
        else if (c3b_records_check_device(c3b_records_view(core, opt), in_check, stream, &fault)) return 1;
        if (on_device && c3b_records_pairs(opt) < fault) fault = c3b_records_pairs(opt);
        if (fault != C3B_REC_OK) {
            c3b_set_error("%s: records: read %lld: %s", who, (long long)c3b_records_fault_read(fault), c3b_records_fault_text(fault));
            return 1;
        }
        C3bReads r{};
        r.n = n;
        int64_t nc = 0, ns = 0;
        if (n > 0) {
            // the check has held each closing offset to its count
            nc = core->n_cigar;
            ns = core->n_seq;
            const int64_t nq = opt ? opt->n_qual : 0, nn = opt ? opt->n_qname : 0, nm = opt ? opt->n_mv : 0;
            const size_t n0 = (size_t)n, n1 = (n0 + 1) * 8;
            auto up = [&](C3bBuf &b, const auto *src, size_t bytes, auto &dev) {
                return c3b_upload(b, src, bytes, on_device, dev, stream, who);
            };
            if (up(in_core[0], core->pos, n0 * 8, r.pos) || up(in_core[1], core->flag, n0 * 2, r.flag) ||
                up(in_core[2], core->mapq, n0, r.mapq) || up(in_core[3], core->cigar_off, n1, r.cigar_off) ||
                up(in_core[4], core->cigar, (size_t)nc * 4, r.cigar) || up(in_core[5], core->seq_off, n1, r.seq_off) ||
                up(in_core[6], core->seq, (size_t)ns, r.seq) || up(in_core[7], core->l_qseq, n0 * 4, r.l_qseq))
                return 1;
            if (opt && opt->qual_off && (up(in_qoff, opt->qual_off, n1, r.qual_off) || up(in_qual, opt->qual, (size_t)nq, r.qual)))
                return 1;
            if (opt && opt->qname_off &&
                (up(in_noff, opt->qname_off, n1, r.qname_off) || up(in_name, opt->qname, (size_t)nn, r.qname)))
                return 1;
            if (opt && opt->mv_off && want_mv && (up(in_moff, opt->mv_off, n1, r.mv_off) || up(in_mv, opt->mv, (size_t)nm * 4, r.mv)))
                return 1;
        }
        const char *d = nullptr;
        if (c3b_upload(in_ref, ref_seq, (size_t)(ref_len > 0 ? ref_len : 0), on_device, d, stream, who)) return 1;
        R = r;
        dref = d;
        this->ref_start = ref_start;
        this->ref_len = ref_len > 0 ? ref_len : 0;
        n_cigar = nc;
        n_seq = ns;
        return 0;
    }

    // The text stage over up to n candidates (the counter's region width, the builder's candidate count): sizes and grows its
    // buffers from what the host knows when the stage is enqueued, and fills the arguments both stages share.  `what` names
    // the owner in allocation errors.
    int text_prepare(int64_t n, int64_t max_indel_length, const char *what, C3bAltText &t) {
        C3B_CUDA(cudaSetDevice(device));
        texted = false;
        // every allele record comes from one insertion / deletion operation of one read
        const int64_t cap = n_cigar < C3B_AL_CAP ? (n_cigar > 0 ? n_cigar : 1) : C3B_AL_CAP;
        // bytes: head, SNP and R fields per candidate; key, count and separators per record; the inserted bases are query bases;
        // a printed deletion shows at most max_indel_length reference bases
        const int64_t del_len = max_indel_length < 0 ? 0 : (max_indel_length < ref_len ? max_indel_length : ref_len);
        const int64_t del_bytes = cap * del_len < (1ll << 28) ? cap * del_len : (1ll << 28);
        const int64_t text_cap = 160 * (n + 1) + 48 * cap + 2 * n_seq + del_bytes;
        const size_t nz = (size_t)n + 1;
        auto grow = [&](C3bBuf &b, size_t bytes) { return b.ensure(bytes, stream, what); };
        if (grow(tx_hash, (size_t)cap * 4) || grow(tx_order, (size_t)cap * 4) || grow(tx_table, (8 * nz + 3 * (size_t)cap) * 4) ||
            grow(tx_nins, nz * 4) || grow(tx_ndel, nz * 4) || grow(tx_len_text, nz * 4) || grow(tx_len_dec, nz * 4) ||
            grow(tx_text, (size_t)text_cap) || grow(tx_dec, (size_t)text_cap) || grow(tx_text_off, nz * 8) ||
            grow(tx_dec_off, nz * 8) || grow(tx_ref_base, nz) || grow(tx_position, nz * 8))
            return 1;
        int64_t *cnt = counters.as<int64_t>();
        t.n = n; t.ref_start = ref_start; t.ref_len = ref_len; t.max_indel_length = max_indel_length;
        t.ref = dref; t.R = R;
        t.al_off = al_off.as<int32_t>(); t.al_n = al_n.as<int32_t>();
        t.al_meta = al_meta.as<uint32_t>(); t.al_read = al_read.as<uint32_t>(); t.al_qpos = al_qpos.as<uint32_t>();
        t.al_cnt = al_cnt.as<uint32_t>(); t.al_cap = cap;
        t.hash = tx_hash.as<uint32_t>(); t.order = tx_order.as<int32_t>(); t.table = tx_table.as<uint32_t>();
        t.n_ins = tx_nins.as<int32_t>(); t.n_del = tx_ndel.as<int32_t>();
        t.len_text = tx_len_text.as<int32_t>(); t.len_dec = tx_len_dec.as<int32_t>();
        t.status = reinterpret_cast<int *>(cnt + text_word);
        t.text = tx_text.as<char>(); t.dec = tx_dec.as<char>(); t.text_cap = t.dec_cap = text_cap;
        t.text_off = tx_text_off.as<int64_t>(); t.dec_off = tx_dec_off.as<int64_t>(); t.totals = cnt + text_word + 1;
        t.ref_base = tx_ref_base.as<uint8_t>(); t.position = tx_position.as<int64_t>();
        return 0;
    }
    // Queues the stage text_prepare sized: clears its three counter words (an earlier stage's overflow is not this one's), runs
    // launch(a, stream, launches) between the stage's events, and copies the counter block back, so the workspace's next wait
    // also brings the stage's status and byte totals.
    template <class Args> int text_enqueue(const Args &a, int (*launch)(const Args &, cudaStream_t, int *)) {
        launches[1] = 0;
        C3B_CUDA(cudaMemsetAsync(counters.as<int64_t>() + text_word, 0, 3 * 8, stream));
        C3B_CUDA(cudaEventRecord(ev[1][0], stream));
        if (launch(a, stream, &launches[1])) return 1;
        C3B_CUDA(cudaEventRecord(ev[1][1], stream));
        C3B_CUDA(cudaMemcpyAsync(host_counters, counters.p, (size_t)n_counters * 8, cudaMemcpyDeviceToHost, stream));
        texted = true;
        return 0;
    }
    // The stage's byte totals, once the workspace's own wait has brought the counter block.  `who` names the entry point in the
    // error, `hint` what its caller can do when the text outgrew the stage's buffers.
    int text_sizes(const char *who, const char *hint, int64_t *n_text_bytes, int64_t *n_decoder_bytes) {
        if (host_counters[text_word] != 0) {
            c3b_set_error("%s: the all_alt_info text outgrew its buffers; %s or lower max_indel_length", who, hint);
            return 1;
        }
        if (n_text_bytes) *n_text_bytes = host_counters[text_word + 1];
        if (n_decoder_bytes) *n_decoder_bytes = host_counters[text_word + 2];
        return 0;
    }
    // Copies the stage's outputs for n_cand candidates into whichever host arrays are given, and waits for them.
    int text_fetch(const char *who, const char *hint, int64_t n_cand, char *text, int64_t *text_off, char *decoder,
                   int64_t *decoder_off, uint8_t *ref_base, int64_t *position) {
        int64_t nt = 0, nd = 0;
        if (text_sizes(who, hint, &nt, &nd)) return 1;
        const size_t nk = (size_t)n_cand;
        return get(text, tx_text, (size_t)nt) || get(text_off, tx_text_off, (nk + 1) * 8) || get(decoder, tx_dec, (size_t)nd) ||
               get(decoder_off, tx_dec_off, (nk + 1) * 8) || get(ref_base, tx_ref_base, nk) || get(position, tx_position, nk * 8) ||
               wait();
    }
    // The stage's outputs where they live on the device.
    void text_device(const char **text, const int64_t **text_off, const char **decoder, const int64_t **decoder_off,
                     const uint8_t **ref_base, const int64_t **position) const {
        if (text) *text = tx_text.as<char>();
        if (text_off) *text_off = tx_text_off.as<int64_t>();
        if (decoder) *decoder = tx_dec.as<char>();
        if (decoder_off) *decoder_off = tx_dec_off.as<int64_t>();
        if (ref_base) *ref_base = tx_ref_base.as<uint8_t>();
        if (position) *position = tx_position.as<int64_t>();
    }
};

// Creates a W (derived from C3bRegionWorkspace) on device `ordinal`: `stages` event pairs and a block of `n_counters` int64
// counters, on the device and pinned on the host, of which `text_word` and the two after it are the text stage's.  `who` names
// the entry point in the errors.
template <class W> int c3b_region_create(W **out, int ordinal, int stages, int n_counters, int text_word, const char *who) {
    if (!out) { c3b_set_error("%s: null out", who); return 1; }
    *out = nullptr;
    if (c3b_use_device(ordinal, 1, nullptr)) return 1;
    W *w = new W();
    w->device = ordinal;
    w->n_counters = n_counters;
    w->text_word = text_word;
    bool ok = w->counters.ensure((size_t)n_counters * 8, nullptr, who) == 0 &&
              cudaMallocHost((void **)&w->host_counters, (size_t)n_counters * 8) == cudaSuccess;
    for (int i = 0; i < stages && ok; ++i)
        ok = cudaEventCreate(&w->ev[i][0]) == cudaSuccess && cudaEventCreate(&w->ev[i][1]) == cudaSuccess;
    if (!ok) {
        c3b_set_error("%s: event / pinned allocation failed", who);
        delete w;
        return 1;
    }
    *out = w;
    return 0;
}

// Releases a workspace on its own device.
template <class W> void c3b_region_destroy(W *w) {
    if (!w) return;
    cudaSetDevice(w->device);
    delete w;
}

struct HostParam {
    std::vector<float> data;
    std::vector<int64_t> shape;
};

// One dense head: L5_k (D4 -> 128) then Y_k (128 -> n).  fp32, transposed for coalesced reads.
struct HeadWeights {
    const float *w5t;   // [D4][128]
    const float *b5;    // [128]
    const float *by;    // [n]
    int n;
    int out_off;
};

struct HeadsParams {
    HeadWeights h[C3B_MAX_HEADS];
    const float *b4;    // [D4]
    const float *wy_all; // [128][out_dim]: every head's output weights side by side (column = global output index)
    int nheads;
    int d4;
    int out_dim;
};

// ---- fp32 debug path weights (device pointers) ----
struct LstmF32 {
    const float *wih_t;  // [I][4H]
    const float *whh_t;  // [H][4H]
    const float *bias;   // [4H] = b_ih + b_hh
};
struct ConvF32 {
    const float *w;      // [9][Cin][Cout]  (BN folded; conv1 also carries 1/100)
    const float *bias;   // [Cout]          (BN folded)
    int cin, cout, stride;
};

// ---- tensor-core path packed operands (device pointers into weight image 0) ----
struct IgemmW {
    const op_t *w_img;   // wgmma B-operand image per k-chunk: [nchunks][8 kgroups][N rows][8] fp16
    const float *bias;            // [N]
    int n;                        // output columns (Cout / gate rows / dense units)
    int kgroups;                  // K/8 (16-byte k-groups), real
    int nchunks;                  // ceil(kgroups/8)
};

// Zero-padded channel-group-planar feature map [C/8][p][8]: slot(b,h,w) = g + b*s + (h+1)*wp + (w+1)  (see pconv_tc.cu)
struct PlanarGeom {
    int h, w, wp, s, g;        // real dims, padded width (w+2), slots per site ((h+2)*wp), guard slots
    int64_t t, p;              // data slots (B*s), plane pitch in slots (g + roundup(t,512) + g)
};
// `cap` >= batch: the site count the plane pitch is laid out for (a workspace keeps the layout of its largest chunk, so smaller
// chunks find their borders / guards already zero)
inline PlanarGeom c3b_planar_geom(int64_t batch, int h, int w, int64_t cap = 0) {
    PlanarGeom g;
    g.h = h; g.w = w; g.wp = w + 2; g.s = (h + 2) * (w + 2);
    g.g = (g.wp + 1 + 7) / 8 * 8;
    g.t = batch * g.s;
    const int64_t tc = (cap > batch ? cap : batch) * g.s;
    g.p = g.g + (tc + 511) / 512 * 512 + g.g;
    return g;
}

// Debug tap: where an intermediate activation of the last forward lives and how to unpack it (c3b_get_tap, option "taps")
struct Tap {
    const void *ptr;
    int fmt;        // 0 f32, 1 fp16
    int layout;     // 0 [B][inner] row-major; 2 k-group-planar [inner/8][bp][8] (row = site);
                    // 3 k-group-planar time-major [inner/8][33*bp][8] (row = t*bp + site) -> [B][33][inner]
                    // 4 zero-padded planar feature map [inner/8][geom.p][8] -> NHWC [B][h][w][inner]
                    // 7 row-major time-major [33*bp][inner] (row = t*bp + site) -> [B][33][inner]
    int64_t inner;
    int bp;
    PlanarGeom geom;
    int nsplit = 1;  // layout 5: [nsplit][bp][inner] split-K partial sums -> summed [B][inner]
    int h = 0, w = 0;  // layout 6: four parity planes [4][inner/8][geom.p][8] (geom = NEXT level) of an h x w map -> NHWC
};

struct Workspace {
    cudaStream_t stream = nullptr;
    C3bBuf dev{C3bBuf::exact};       // device scratch, carved by the forward pass
    C3bBuf stage{C3bBuf::exact};     // host arguments of a call (Staging in c3b_api.cu), after stage 3's kernel scratch
    // full-alignment planar maps are laid out for `fa_cap_sites` sites (the largest chunk seen on this workspace); smaller
    // chunks reuse that layout (their borders / guards are already zero), so a ragged tail never re-clears the region
    int64_t fa_cap_sites = 0;
    int fa_cap_depth = -1;
    bool fa_zeroed = false;
    std::map<std::string, Tap> taps;   // per workspace, filled only while option "taps" is on
    // per-kernel CUDA-event pairs recorded while option "profile" is on (resolved lazily by c3b_get_profile)
    struct ProfRec { const char *name; cudaEvent_t e0, e1; long long ctas; };
    std::vector<ProfRec> prof;
};

struct c3b_model {
    int kind = 0, channels = 0, add_indel = 0, device = 0;
    int nheads = 2, out_dim = 24, d4 = 128, l4_in = 0;
    int precision = C3B_PREC_F16_TC;
    int chunk_sites = 0;
    int lstm_tile = 0;
    int profile = 0;
    int lstm_wg = 2;                   // warpgroups (one sub-tile of sites each) per LSTM CTA (option "lstm_wg": 1 or 2)
    int lstm2_split = 1;               // LSTM2 split by block pair (option "lstm2_split"): 1 lstm2_split_kernel at 32 sites at most;
                                       // 2 the same kernel at 48 sites where LSTM1 runs 64-site tiles; 0 the sub-tile kernel
    int lstm_mufu16 = 0;               // 1: packed tanh.approx.f16x2 gate activations, 0 (default, faster: the epilogue is issue-bound): fp32 tanh.approx
    int tap_ws = -1;                   // debug: workspace index c3b_get_tap reads
    int taps = 0;                      // debug option "taps": record where the intermediate activations of a forward live
    bool weights_by_broadcast = false; // the packed images arrived by c3b_bcast_weights (no host-side parameters behind them)
    long long *lstm_trace = nullptr;   // device [2][33][4] clock stamps (debug option "lstm_trace")
    std::map<std::string, std::pair<double, int64_t>> prof_total;   // name -> (ms, launches)
    std::map<std::string, double> prof_ctas;                         // name -> sum of CTAs launched
    int sm_count = 132;
    bool finalized = false;
    std::map<std::string, HostParam> params;
    std::vector<std::string> expected;
    std::map<std::string, std::vector<int64_t>> expected_shape;

    // device weights, the units c3b_weight_blob exposes and c3b_bcast_weights sends: image 0 holds everything the tensor-core
    // forward reads, image 1 what only the fp32 path reads (the fp32 path reads both)
    C3bBuf blob{C3bBuf::exact};      // image 0
    C3bBuf f32blob{C3bBuf::exact};   // image 1

    HeadsParams heads;                 // image 0, read by both paths
    // fp32 path, image 1
    LstmF32 lstm_f32[2][2];
    const float *l4_f32_t = nullptr;   // [l4_in][d4]
    ConvF32 conv_f32[9];
    // tc path, image 0
    // LSTM1 / LSTM2 wgmma A-operand image, both directions: [dir][2H/64 blocks][K/8][64 rows][8] fp16, rows permuted
    // (c3b_lstm_row).  LSTM1's bias is a weight column against the constant-1 input; LSTM2's rides in the projection.
    const op_t *lstm_tc[2] = {};
    IgemmW proj2;                      // LSTM2 input projection, both directions: N = 1280 (column order c3b_lstm2_pg_row)
    const op_t *l4_tc = nullptr;       // L4 B-operand image (tail_tc.cu): [l4_in/64 chunks][8 kg][d4 rows][8]
    IgemmW conv_tc[9];

    std::vector<Workspace *> ws;
    int64_t launches = 0;
    int64_t last_batch = 0;
};

// conv order used everywhere: 0 conv1, 1 rb1.conv1, 2 rb1.conv2, 3 conv3, 4 rb2.conv1, 5 rb2.conv2, 6 conv5, 7 rb3.conv1, 8 rb3.conv2

// ---- kernels_common.cu ----
int c3b_launch_ingest_pileup_f32(const void *x, int dtype, float *out, int64_t n_elems, cudaStream_t s);
int c3b_launch_ingest_fa_f32(const void *x, int dtype, float *out, int64_t n_elems, cudaStream_t s);
// z4: nsplit partial sums [nsplit][split_stride] of the L4 pre-activation (no bias); the kernel adds them
int c3b_launch_heads(const float *z4, int nsplit, int64_t split_stride, const HeadsParams &hp, float *out, int64_t batch, cudaStream_t s);

// ---- decode.cu ----
int c3b_launch_decode_stage1(const float *y, const uint8_t *ref_gt21, int64_t batch, int out_dim, uint8_t *is_ref, float *ref_prob,
                             int32_t *argmax, float *maxprob, double *qual, int32_t *nonref_idx, int32_t *n_nonref, cudaStream_t s);
// sites == nullptr: site s is row s; n_sites == nullptr: max_sites sites (else min(*n_sites, max_sites), read on the device)
int c3b_launch_decode_stage2(const float *y, const uint8_t *ref_gt21, int64_t batch, int out_dim, const int32_t *sites,
                             const int32_t *n_sites, int64_t max_sites, int k, uint8_t *cat, uint16_t *idx, float *prob,
                             uint16_t *tie_mask, int32_t *count, uint8_t *complete, cudaStream_t s);

// stage 3 (c3b_decode_calls): stage 1, stage 2 and the walks on device pointers; scratch holds c3b_calls_scratch_bytes()
size_t c3b_calls_scratch_bytes(int64_t batch, int out_dim, int k, int64_t n_alt_bytes);
int c3b_launch_decode_calls(const float *y, const uint8_t *ref_base, int64_t batch, int out_dim, const char *alt_bytes,
                            const int64_t *alt_offsets, int64_t n_alt_bytes, uint32_t cfg, int64_t max_infer_len, int k,
                            c3b_call *calls, char *text, int64_t *ad, void *scratch, cudaStream_t s);

// ---- kernels_fp32.cu ----
int c3b_launch_lstm_f32(const float *x, const LstmF32 &fwd, const LstmF32 &bwd, float *out, int64_t batch, int in_dim,
                        int hidden, cudaStream_t s);
int c3b_launch_dense_f32(const float *x, const float *w_t, float *out, int64_t batch, int k, int n, cudaStream_t s);
int c3b_launch_conv_f32(const float *x, const ConvF32 &w, const float *residual, float *out, int64_t batch, int hin,
                        int win, int hout, int wout, cudaStream_t s);
int c3b_launch_spp_f32(const float *x, float *out, int64_t batch, int h, int w, int c, cudaStream_t s);

// ---- tensor-core path ----
struct TcPileupBuffers {
    op_t *x_tap;  // [33][B][48] fp16, time-major: LSTM1's hi(x) | 1 | lo(x) operand columns; only with the "taps" option, else nullptr
    op_t *h1;     // tile-major k-group-planar, 32 k-groups: row = t*Bp + b, k = dir*128 + j  (projection GEMM operand)
    __half *pg;            // [33*B][1280] fp16 pre-gates of LSTM2 (bias included), column dir*640 + C in gate-quad order (c3b_lstm2_pg_row)
    op_t *h2;     // tile-major k-group-planar, 1320 k-groups: row = b, k = t*320 + dir*160 + j (flatten order of clair3/model.py:135)
    float *z4;             // [16][B][128] fp32 split-K partial sums of the L4 pre-activation (no bias)
    int bp;                // padded batch: multiple of 128
};
// Where a pileup chunk's sites come from: a dense [n,33,C] tensor, or 33-row windows of a per-column count matrix
// ([n_cols][C], libclair3's plp_data.matrix) starting at rows starts[b] (rows outside the matrix, or outside [bounds[b][0],
// bounds[b][1]) when bounds are given, read as zero)
struct PileupSrc {
    const void *x;          // dense: first site of the chunk; windows: the column matrix
    int dtype;
    const int64_t *starts;  // windows: device pointer to this chunk's first start row; nullptr = dense
    const int64_t *bounds;  // windows: device pointer to this chunk's first [lo, hi) row pair; nullptr = [0, n_cols)
    int64_t n_cols;
};
int c3b_launch_gather_windows_f32(const void *cols, int dtype, int channels, const int64_t *starts, const int64_t *bounds,
                                  int64_t n_cols, float *out, int64_t batch, cudaStream_t s);
int c3b_launch_proj2(const c3b_model *m, const op_t *h1, const IgemmW &w, __half *pg, int bp, cudaStream_t s);
int c3b_launch_tail(const c3b_model *m, const op_t *act, int64_t batch, int bp, float *out, float *z4, int *nsplit_out, cudaStream_t s);
// LSTM1 reads the chunk's `batch` sites straight from src and builds its x operand columns itself
int c3b_launch_lstm1_tc(const c3b_model *m, const TcPileupBuffers &b, const PileupSrc &src, int64_t batch, int tile,
                        cudaStream_t s);
int c3b_launch_lstm2_tc(const c3b_model *m, const TcPileupBuffers &b, int64_t batch, int tile, bool split, cudaStream_t s);

struct PconvArgs {
    const op_t *in;            // planar padded, c channels
    op_t *out;                 // planar padded, n channels, same geometry
    const op_t *residual;      // optional, planar padded like out
    IgemmW w;                  // per-chunk weight images (k = tap*c + ci)
    PlanarGeom geom;           // geometry of the OUTPUT level (= input level for stride 1)
    int c, n, relu;
    int stride2;               // 1: `in` holds the four parity planes of the previous level, each [c/8][geom.p][8] (see pconv_tc.cu)
    int out_parity;            // 1: `out` receives the real pixels scattered into the four parity planes of `next` ([n/8][next.p][8] each)
    PlanarGeom next;
};
// offset (elements) of padded pixel (hp, wp) of site b, channel group 0, inside a parity-plane set of geometry g with c channels
inline size_t c3b_parity_offset(const PlanarGeom &g, int c, int64_t b, int hp, int wp) {
    return (size_t)((hp & 1) * 2 + (wp & 1)) * ((size_t)(c / 8) * g.p * 8) + ((size_t)g.g + b * g.s + (size_t)((hp >> 1) + 1) * g.wp + ((wp >> 1) + 1)) * 8;
}
int c3b_launch_pconv(const c3b_model *m, const PconvArgs &a, cudaStream_t s);

int c3b_launch_ingest_fa_tc(const void *x, int dtype, int channels, int cpad, op_t *out, int64_t batch, int depth, const PlanarGeom &g1,
                            cudaStream_t s);
int c3b_launch_spp_tc(const op_t *x, const PlanarGeom &g, op_t *out, int64_t batch, int c, int bp, cudaStream_t s);

// ---- pileup feature counter: the all_alt_info text stage (plp_alt_text.cu), enqueued by c3b_plp_alt_text in plp_counts.cu ----
// n is the region's width, end - start; the candidates are the count's, their number a device counter
struct PlpAltTextArgs : C3bAltText {
    int64_t start, end;
    const int64_t *n_cand;              // device counter
    const int64_t *cand_cols, *major, *matrix;
    const int32_t *stats, *ins_last;
    int32_t *mate;                      // scratch [al_cap]
};
int c3b_launch_plp_alt_text(const PlpAltTextArgs &a, cudaStream_t s, int *launches);

// ---- full-alignment builder: the all_alt_info text stage (fa_alt_text.cu), enqueued by c3b_fa_alt_text in fa_tensor.cu ----
// n is the number of candidates, known on the host
struct FaAltTextArgs : C3bAltText {
    const int64_t *cand;                // [n] 0-based positions
    const int32_t *c_depth, *c_acgt;
};
int c3b_launch_fa_alt_text(const FaAltTextArgs &a, cudaStream_t s, int *launches);
