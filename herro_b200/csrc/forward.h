// forward.h — device-resident weights of the forward stage (see herro_b200/weights.py for the
// blob format and tensor names).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <vector>
#include "common.cuh"

namespace hb {

constexpr int MAX_LAYERS = 8;

struct SplitW {  // bf16 hi / lo split of an fp32 weight matrix [N,K] (gemm_tc.cu)
    const void *hi = nullptr, *lo = nullptr;
};

struct FwdLayer {
    const float *ln1_g, *ln1_b, *wqkv, *bqkv, *wo, *bo, *ln2_g, *ln2_b, *w1, *b1, *w2, *b2;
    SplitW s_qkv, s_o, s_1, s_2;
    SplitW s_qkvp;               // Wqkv with rows regrouped per head [H][q(32) | k(32) | v(32)][C] (fused QKV+attention kernel)
    const float* bqkvp = nullptr;  // bqkv in the same order; nullptr: fused kernel unavailable
};

struct PosLayer {  // an encoder layer of the position-axis stage (width D, pos_heads heads, pos_ffn hidden)
    const float *ln1_g, *ln1_b, *bqkv, *bo, *ln2_g, *ln2_b, *b1, *b2;
    SplitW s_qkv, s_o, s_1, s_2;
};

struct FwdWeights {
    int stem_k, C, H, layers, F, D;
    const float* stem_tab;  // [K][12][C]  = sum_e stem_w[c][e][j] * emb[t][e]   (embedding folded into the conv)
    const float* stem_wq;   // [K][C]      = stem_w[c][6][j]                     (quality channel)
    const float* stem_b;    // [C]
    const float* read_pos;  // [31][C]
    FwdLayer layer[MAX_LAYERS];
    const float *lnf_g, *lnf_b, *wc, *bc, *wb, *bb, *wi, *bi;
    SplitW s_c;
    SplitW s_stem;          // W' of the tensor-core stem, [C][stem_kp]
    int stem_kblocks = 0;   // 0: tensor-core stem unavailable (C != 128 or too many taps)
    int num_sms;
    // debugging aids / A-B parity tests, read from the environment ONCE in hb_create (HERRO_B200_NO_FUSE_{LN,FFN,ATTN})
    int no_fuse_ln = 0, no_fuse_ffn = 0, no_fuse_attn = 0, no_fuse_oproj = 0;
    // position-axis encoder stage after the collapse (0 layers: none); kept last so the fields above keep their offsets
    int pos_layers = 0, pos_heads = 0, pos_ffn = 0;
    PosLayer pos[MAX_LAYERS];
};

// gemm_tc.cu
enum { GEMM_OUT_F32 = 0, GEMM_OUT_F32_RELU = 1, GEMM_OUT_F32_RES = 2, GEMM_OUT_SPLIT_RELU = 3,
       GEMM_OUT_F32_RES_LN = 4 /* N == 128: out = acc+bias+res (fp32) and LayerNorm(out) as split bf16 */ };
struct GemmArgs {
    const __nv_bfloat16 *Ahi, *Alo;  // activations, split bf16, row stride lda (elements)
    size_t lda;
    const __nv_bfloat16 *Whi, *Wlo;  // weights [N,K], split bf16
    uint32_t K;
    const float* bias;               // [N]
    float* out;                      // fp32 output (modes F32*), row stride ldc
    const float* res;                // residual (mode F32_RES), same layout as out
    size_t ldc;
    __nv_bfloat16 *out_hi, *out_lo;  // split bf16 output (mode SPLIT_RELU), row stride ldo
    size_t ldo;
    const float *ln_g, *ln_b;        // LayerNorm affine (mode F32_RES_LN)
    uint32_t m_tiles, n_chunks, k_blocks;  // M/128, N/128, K/64
    int mode;
};
struct FfnArgs {  // k_ffn_ws: fused FFN for C == 128, F == 512
    const __nv_bfloat16 *Hhi, *Hlo;        // LayerNorm(X), split bf16, [T][128]
    const __nv_bfloat16 *W1hi, *W1lo;      // [F][128]
    const __nv_bfloat16 *W2hi, *W2lo;      // [128][F]
    const float *b1, *b2;                  // [F], [128]
    float* X;                              // residual stream [T][128], updated in place
    const float *ln_g, *ln_b;              // LayerNorm that follows
    __nv_bfloat16 *out_hi, *out_lo;        // LayerNorm(X_new), split bf16, [T][128]
    uint32_t F, m_tiles;
    // fused attention out-projection (k_ffn_ws<true>): Hhi/Hlo then hold the attention output O, and the kernel first computes
    // X += O · Wo^T + bo, H = LayerNorm(X; ln2) on chip.  Wohi == nullptr: unfused (H is read as given).
    const __nv_bfloat16 *Wohi = nullptr, *Wolo = nullptr;  // [128][128]
    const float *bo = nullptr, *ln2_g = nullptr, *ln2_b = nullptr;
    int store_x = 1;  // 0: do not write the updated residual stream back (last layer: only LayerNorm(X) is consumed)
};
cudaError_t ffn_tc(const FfnArgs& a, int num_sms, cudaStream_t st);
struct QkvAttnArgs {  // k_qkv_attn_ws: QKV projection + read-axis attention for C == 128, 4 heads
    const __nv_bfloat16 *Hhi, *Hlo;      // LayerNorm(X), split bf16, [T][128]
    const __nv_bfloat16 *Whi, *Wlo;      // head-grouped Wqkv [4*96][128]
    const float* bias;                   // head-grouped bqkv [4*96]
    __nv_bfloat16 *out_hi, *out_lo;      // attention output, split bf16, [T][128] (may alias Hhi/Hlo: tile-local in-place)
    uint32_t m_tiles;
};
cudaError_t qkv_attn_tc(const QkvAttnArgs& a, int num_sms, cudaStream_t st);
struct StemArgs {  // k_stem_tc: the stem as a contraction over taps x 16 features (C == 128 only)
    const __nv_bfloat16 *Whi, *Wlo;  // W' [128][Kp], split bf16
    uint32_t Kp;                     // k_blocks * 64
    uint32_t k_blocks, taps;
    const float *bias, *read_pos;    // [128], [31][128]
    float* X;                        // [positions*32][128]
    uint32_t n0, npos;               // work-list range
    const float *ln_g = nullptr, *ln_b = nullptr;          // optional: LayerNorm(X) of every row, emitted as split bf16
    __nv_bfloat16 *out_hi = nullptr, *out_lo = nullptr;    // [positions*32][128]; nullptr: X only
};
cudaError_t stem_tc(const BatchView& b, const StemArgs& a, int num_sms, cudaStream_t st);
// pos_attn.cu: attention over variable-length sequences of rows (sequence i = rows [seq_base[i] - base_sub, + seq_len[i])
// of `qkv`, whose row holds q | k | v, D each, heads of D / heads in {32, 64}); keys past a sequence's length are masked.
// Writes the attention output of each sequence row as split bf16; rows outside every sequence are not written.
struct PosAttnArgs {
    const float* qkv;                // [rows][ld_qkv] fp32
    size_t ld_qkv;
    const uint64_t* seq_base;        // [n_seq]
    const uint32_t* seq_len;         // [n_seq]
    uint64_t base_sub;
    uint32_t n_seq;
    int D, heads;
    __nv_bfloat16 *out_hi, *out_lo;  // [rows][ldo]
    size_t ldo;
};
cudaError_t pos_attention(const PosAttnArgs& a, cudaStream_t st);
// Z[n] += sinusoidal encoding of the index of position n0 + n within its window, n < npos (Z: [npos][D] fp32)
void launch_pos_embed(const BatchView& b, uint32_t n0, uint32_t npos, int D, float* Z, cudaStream_t st);
cudaError_t split_weights(const float* w, size_t n, void** hi, void** lo);
cudaError_t gemm_tc(const GemmArgs& a, int num_sms, cudaStream_t st);
// forward.cu (fp32 SIMT contraction: the self test's reference)
void gemm_simt(int act, int res, const float* A, int lda, const float* Wt, const float* bias, float* Cout, int ldc,
               const float* Res, size_t M, int N, int K, cudaStream_t st);

// Per-kernel-class CUDA-event timing on the launching stream (off during replays).
struct KTimer {
    bool on = false;
    cudaStream_t st = nullptr;
    std::vector<cudaEvent_t> pool;
    size_t used = 0;
    struct Rec { int cls; size_t e0, e1; };
    std::vector<Rec> recs;
    uint64_t launches[16] = {0};
    cudaEvent_t get() {
        if (used == pool.size()) { cudaEvent_t e; cudaEventCreate(&e); pool.push_back(e); }
        return pool[used++];
    }
    void begin(int cls) {
        launches[cls]++;
        if (!on) return;
        recs.push_back(Rec{cls, used, used + 1});
        cudaEventRecord(get(), st);
        get();
    }
    void end() {
        if (!on) return;
        cudaEventRecord(pool[recs.back().e1], st);
    }
    // after the stream is synchronised: add elapsed ms per class, reset
    void collect(double* ms, uint64_t* n) {
        for (auto& r : recs) { float t = 0; cudaEventElapsedTime(&t, pool[r.e0], pool[r.e1]); ms[r.cls] += t; }
        for (int i = 0; i < 16; i++) { n[i] += launches[i]; launches[i] = 0; }
        recs.clear();
        used = 0;
    }
    void discard() { for (auto& l : launches) l = 0; recs.clear(); used = 0; }
    void destroy() { for (auto e : pool) cudaEventDestroy(e); pool.clear(); }
};
enum { K_TOKENIZE = 0, K_PASS1, K_SCORES, K_PASS2A, K_SCAN, K_PILEUP, K_LISTS, K_STEM, K_LAYERNORM, K_GEMM, K_ATTENTION,
       K_HEADS, K_CONSENSUS, K_FFN, K_QKV_ATTN, K_POS_ATTN };

// Scratch is carved from one allocation into arrays that each start 256-byte aligned, the alignment a separate cudaMalloc
// would give: TMA operands and 16-byte row stores rely on it.
inline size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }
size_t fwd_workspace_bytes(const FwdWeights& wt, uint32_t chunk_pos);
// Runs positions [n0, n0+npos) of the work list: whole windows [w0, w0+nwin) (the position-axis stage attends within them)
int launch_forward_chunk(const BatchView& b, const FwdWeights& wt, uint32_t n0, uint32_t npos, uint32_t w0, uint32_t nwin,
                         uint8_t* ws, float* logits, float* info, cudaStream_t st, KTimer& kt);
uint64_t forward_flops_per_pos(const FwdWeights& wt, uint64_t* gemm_flops);
// FLOPs of the position-axis attention (QK^T and PV) of windows with the given supported-position counts
uint64_t pos_attn_flops(const FwdWeights& wt, const uint32_t* nsup, size_t nwin);
// algorithmic FLOPs per supported position attributed to the kernel class that executes them on the active code path
void forward_class_flops_per_pos(const FwdWeights& wt, uint64_t (&out)[16]);

// batch_in.cu: a caller's [rows][31] tokens and quality bytes (any alignment) -> the [rows][32] matrices, column 31 = token 10 /
// quality 33; a token above 11 is written as 0xff (contributes nothing) and the smallest linear index of one is atomicMin'ed into *bad
void launch_batch_in(const uint8_t* tok, const uint8_t* qual, uint64_t rows, uint8_t* mat_b, uint8_t* mat_q, unsigned long long* bad,
                     cudaStream_t st);

// cons_in.cu: a caller's ConsensusWindows -> row_emit (class 0..4 | 0x80 if supported) of every row of the windows with
// n_alns >= 2, at w_rowbase; the smallest linear byte index of a token the reference's consensus() would panic on is atomicMin'ed
// into *bad
struct ConsInArgs {
    const uint8_t* tok;          // [rows][31] BASES_MAP tokens, window after window, any alignment
    const float* logits;         // [supported][5]
    const uint2* keys;           // per window from w_keybase: (pos << 8 | ins, logit row), sorted by key, unique
    const uint32_t* w_L;         // rows
    const uint32_t* w_nsel;      // n_alns
    const uint64_t* w_rowbase;   // first row
    const uint64_t* w_keybase;   // first key
    const uint32_t* w_nkeys;
    uint8_t* row_emit;
    unsigned long long* bad;
};
void launch_cons_in(const ConsInArgs& a, uint32_t n_win, cudaStream_t st);

// feat_out.cu: the outputs of hb_features_batch.  A RowSeg is `total` output rows from out_row on: the first `valid` are the
// arena's rows from src_row on, the rest padding (token 11 / quality 126).  A ListSeg puts window `win`'s supported list at entry
// sup_out of (pos, ins) / indices and its surviving overlaps' query reads at entry id_out of ids.  Any output may be NULL.
struct RowSeg { uint64_t out_row, src_row; uint32_t valid, total; };
struct ListSeg { uint32_t win, pad; uint64_t sup_out, id_out; };
void launch_rows_out(const RowSeg* seg, uint32_t n_seg, const uint8_t* mat_b, const uint8_t* mat_q, uint8_t* out_b, uint8_t* out_q,
                     cudaStream_t st);
void launch_lists_out(const BatchView& b, const ListSeg* seg, uint32_t n_seg, uint32_t* sup, int32_t* idx, uint32_t* ids, cudaStream_t st);

// reads_in.cu: a launch's reads from the host read store (device-mapped host memory) into its batch region.  The region's arrays
// keep the uploaded store's padding: `words` is READS_FRONT_WORDS zero words, n_words gathered words, READS_BACK_WORDS zero words;
// `qual` likewise in bytes of 33.  Every offset is in words / bytes from the first gathered one, and 16-byte aligned: in the store
// and in the region each read takes its words and qualities rounded up to 16 bytes.
constexpr uint32_t READS_FRONT_WORDS = 32, READS_BACK_WORDS = 8, READS_FRONT_QUAL = 256, READS_BACK_QUAL = 16;
struct ReadCopy { uint64_t src_w, src_q, dst_w, dst_q; uint32_t rid, len; };
struct ReadsInArgs {
    const ReadCopy* list;
    uint32_t n;
    const uint64_t* src_words;        // the store's words and qualities (device-mapped pointers)
    const uint8_t* src_qual;
    uint64_t* words;                  // the region's padded arrays
    uint8_t* qual;
    uint64_t n_words, n_qual;
    uint64_t *word_off, *qual_off;    // [n_reads + 1], written for the listed reads only
};
uint64_t launch_reads_in(const ReadsInArgs& a, cudaStream_t st, KTimer& kt);

// features.cu
cudaError_t features_configure(uint32_t W);
int launch_features_a(const BatchView& b, cudaStream_t st, KTimer& kt);
int launch_pileup(const BatchView& b, cudaStream_t st, KTimer& kt, bool v1);
// windowing_dev.cu: extract_windows on the device (parse, boundaries, op-slot scan); returns the number of kernels launched
int launch_windowing(const BatchView& b, cudaStream_t st);
// k_scan_u32 of features.cu
void launch_scan_u32(const uint32_t* in, uint64_t* out, uint32_t n, uint32_t* counters, int total_slot, uint64_t cap, int overflow_slot,
                     cudaStream_t st);
// pileup.cu
cudaError_t pileup_configure();
void launch_pileup_v2(const BatchView& b, cudaStream_t st);
int launch_features_c1(const BatchView& b, cudaStream_t st, KTimer& kt);
int launch_features_c2(const BatchView& b, cudaStream_t st, KTimer& kt);
int launch_consensus(const BatchView& b, cudaStream_t st, KTimer& kt);

}  // namespace hb
