// features.cu — sm_90a kernels for the pileup ("features") and consensus stages.
//
// Reference semantics: src/features.rs:44-722 (extract_features and helpers),
// src/inference.rs:214-268 (token map, target indices), src/consensus.rs:86-227.
// The structure is NOT the reference's: the reference materialises a first-pass
// [L, 1+max(n,30)] matrix per window only to (a) find first-pass supported rows and
// (b) count per-read matches on them, then re-stacks 31 columns and drops all-gap rows.
// Here (DESIGN.md §3):
//   pass 1  works position-major without insertion rows (only base rows feed the ranking,
//           src/features.rs:481-491) and never writes a matrix;
//   pass 2  builds the final [L',31] matrix directly: dropping all-gap rows of the
//           re-stacked matrix (src/features.rs:531-556) is the same as recomputing max_ins
//           over the 31 selected columns only;
//   the second get_supported (src/features.rs:558) and the non-supported branch of
//   consensus (src/consensus.rs:176-217, the majority vote) are evaluated on the tile while
//   it is still in shared memory.
#include "common.cuh"
#include "forward.h"

namespace hb {

// ------------------------------------------------------------------------------------
// K1: tokenise the CIGAR slice of every overlap-window, clip it (App. A.3), prefix-sum the
//     target/query offsets, apply the indel filter and compute calculate_accuracy.
//     One warp per overlap-window.
// ------------------------------------------------------------------------------------
template <bool RAW>  // RAW: the overlap-window came from the device windowing (windowing_dev.cu) and its ops from the raw-op arrays
__global__ void __launch_bounds__(128) k_tokenize(BatchView b) {
    const int lane = threadIdx.x & 31;
    const uint32_t wi = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (wi >= b.n_ow) return;
    DevOW ow = b.ow[wi];
    const DevOverlap ov = b.ovl[ow.ovl];
    if ((ov.raw_base != RAW_NONE) != RAW) return;
    const DevWin win = b.win[ow.win];
    const uint8_t* __restrict__ cg = b.cig + ov.cig_off + ow.csi;
    const int slen = (int)ow.cei - (int)ow.csi;
    uint32_t flags = 0;
    uint32_t nops = 0;
    const uint32_t* __restrict__ rkl = nullptr;
    if (RAW) {
        flags = b.ow_flags[wi];  // OWF_BAD from k_parse_cigars / k_windows
        nops = (flags & OWF_BAD) ? 0u : b.ow_nops[wi];
        ow.op_base = b.op_base_dev + (uint32_t)b.ow_opoff[wi];
        if (lane == 0) b.ow_mut[wi].op_base = ow.op_base;
        rkl = b.raw_kl + ov.raw_base + ow.csi;
        if (nops == 0) flags |= OWF_BAD;
    } else {
        if (slen <= 0 || ow.cei > ov.cig_len) flags |= OWF_BAD;
    }
    if (ow.tstart < win.tstart || ow.tstart >= win.tstart + win.len) flags |= OWF_BAD;
    // query region must lie inside the query read (decode() asserts, src/haec_io.rs:157)
    {
        uint32_t qlen = b.rs.len[ov.qid];
        if (ow.qend < ow.qstart) flags |= OWF_BAD;
        if (!ov.strand) {
            if ((uint64_t)ov.qstart + ow.qend > qlen) flags |= OWF_BAD;
        } else {
            if (ov.qend < ow.qend || ov.qend - ow.qstart > qlen) flags |= OWF_BAD;
        }
    }
    if (!RAW && !(flags & OWF_BAD)) {
        // ---- parse: lanes 0..9 look back, lanes 10..31 are the 22 active bytes of this step
        for (int base = 0; base < slen; base += 22) {
            const int idx = base - 10 + lane;
            const bool inrange = idx >= 0 && idx < slen;
            const int c = inrange ? (int)__ldg(cg + idx) : 0;
            const bool active = lane >= 10 && inrange;
            const bool is_digit = inrange && c >= '0' && c <= '9';
            const bool is_letter = active && !is_digit;
            uint32_t num = 0, mul = 1;
            bool stop = false;
            int ndig = 0;
#pragma unroll
            for (int s = 1; s <= 10; s++) {
                const int pc = __shfl_up_sync(HB_FULL, c, s);
                const bool ok = (lane >= s) && pc >= '0' && pc <= '9';  // bytes outside the slice were loaded as 0
                if (!stop && ok) {
                    num += (uint32_t)(pc - '0') * mul;
                    mul *= 10u;
                    ndig++;
                } else {
                    stop = true;
                }
                // op lengths rarely have more than 3 digits: leave as soon as every letter of this step has its number
                if (s >= 2 && !__any_sync(HB_FULL, is_letter && !stop)) break;
            }
            const uint32_t mask = __ballot_sync(HB_FULL, is_letter);
            if (is_letter) {
                uint32_t kind = (c == 'M') ? OP_M : (c == 'I') ? OP_I : (c == 'D') ? OP_D : 1u;
                // 10 digits could overflow u32 and a longer number would be truncated: both are
                // outside anything an aligner emits; flag them like the other parse errors.
                if (kind == 1u || num == 0 || ndig == 0 || ndig >= 10) flags |= OWF_BAD;
                const uint32_t k = nops + __popc(mask & ((1u << lane) - 1u));
                if (k < (uint32_t)slen / 2u + 1u) b.op_kl[ow.op_base + k] = kind | (num << 2);  // the slice's region holds slen / 2 + 1 ops
                else flags |= OWF_BAD;  // more letters than digits
            }
            nops += __popc(mask);
        }
        // the slice must end on an op letter (CigarIter would index past the end otherwise)
        if (lane == 0) {
            int lc = __ldg(cg + slen - 1);
            if (lc >= '0' && lc <= '9') flags |= OWF_BAD;
        }
        flags = __reduce_or_sync(HB_FULL, flags);
        if (nops == 0) flags |= OWF_BAD;
    }
    __syncwarp();

    uint32_t tcur = ow.tstart - win.tstart, qcur = 0;
    uint32_t sum_i = 0, sum_d = 0, sum_m = 0;
    if (!(flags & OWF_BAD)) {
        // ---- clip (first / last / single op) and prefix-sum offsets
        for (uint32_t k0 = 0; k0 < nops; k0 += 32) {
            const uint32_t k = k0 + lane;
            uint32_t kind = 0, raw = 0, eff = 0;
            if (k < nops) {
                const uint32_t kl = RAW ? rkl[k] : b.op_kl[ow.op_base + k];
                kind = kl & 3u;
                raw = kl >> 2;
                eff = raw;
                if (nops == 1) {
                    if (ow.ceo <= ow.cso) flags |= OWF_BAD;  // assert, src/features.rs:592-597
                    eff = ow.ceo - ow.cso;
                } else if (k == 0) {
                    if (raw <= ow.cso) flags |= OWF_BAD;  // assert, src/features.rs:600-608
                    eff = raw - ow.cso;
                } else if (k == nops - 1) {
                    eff = ow.ceo;
                }
                if (eff == 0) flags |= OWF_BAD;  // "Operation length cannot be 0"
                if ((kind == OP_I || kind == OP_D) && raw > 50) flags |= OWF_LONG_INDEL;  // unclipped (H2)
                // get_max_ins uses the unclipped insertion length (H3); with windows produced by
                // extract_windows an insertion is never clipped and never first.
                if (kind == OP_I && (eff != raw || k == 0)) flags |= OWF_BAD;
            }
            const uint32_t dt = (k < nops && kind != OP_I) ? eff : 0;
            const uint32_t dq = (k < nops && kind != OP_D) ? eff : 0;
            const uint32_t it = warp_incl_scan(dt, lane), iq = warp_incl_scan(dq, lane);
            if (k < nops) {
                b.op_kl[ow.op_base + k] = kind | (eff << 2);
                b.op_t[ow.op_base + k] = tcur + it - dt;
                b.op_q[ow.op_base + k] = qcur + iq - dq;
            }
            sum_i += (k < nops && kind == OP_I) ? eff : 0;
            sum_d += (k < nops && kind == OP_D) ? eff : 0;
            sum_m += (k < nops && kind == OP_M) ? eff : 0;
            tcur += __shfl_sync(HB_FULL, it, 31);
            qcur += __shfl_sync(HB_FULL, iq, 31);
        }
        flags = __reduce_or_sync(HB_FULL, flags);
        sum_i = warp_sum(sum_i);
        sum_d = warp_sum(sum_d);
        sum_m = warp_sum(sum_m);
        if (tcur > win.len) flags |= OWF_BAD;                    // writes past the window
        if (qcur != ow.qend - ow.qstart) flags |= OWF_BAD;       // query_iter would run dry / leave bases
    }
    __syncwarp();

    float acc = 0.f;
    if (!(flags & (OWF_BAD | OWF_LONG_INDEL))) {
        // ---- calculate_accuracy (src/features.rs:585-679): matches over M ops
        const QView qv = make_qview(b.rs, ov, ow);
        const uint64_t* __restrict__ tw = b.rs.words + b.rs.word_off[win.rid];
        uint32_t m = 0;
        for (uint32_t k = lane; k < nops; k += 32) {  // one op per lane, 32 bases per step (packed 2-bit compare)
            const uint32_t kl = b.op_kl[ow.op_base + k];
            if ((kl & 3u) != OP_M) continue;
            const uint32_t eff = kl >> 2, t0 = win.tstart + b.op_t[ow.op_base + k], q0 = b.op_q[ow.op_base + k];
            for (uint32_t i = 0; i < eff; i += 32) {
                const uint32_t len = eff - i;
                const uint64_t mm = mismatch_groups(extract32(tw, t0 + i), qv.chunk(q0 + i), len);
                m += (len >= 32 ? 32u : len) - (uint32_t)__popcll(mm);
            }
        }
        m = warp_sum(m);
        const uint32_t tot = sum_m + sum_i + sum_d;  // m + s + i + d
        acc = __fdiv_rn((float)m, (float)tot);       // src/features.rs:678
    }
    if (lane == 0) {
        b.ow_nops[wi] = nops;
        b.ow_flags[wi] = flags;
        b.ow_acc[wi] = acc;
        b.ow_tend[wi] = tcur;
        if (flags & OWF_BAD) atomicOr(&b.tgt_err[win.tgt], TERR_BAD_INPUT);
    }
}

// ------------------------------------------------------------------------------------------------
// K2: first pass of one window.  filter + stable sort by -accuracy (src/features.rs:376-409),
//     first-pass supported base rows (get_supported on the [L, 1+max(n,30)] matrix, :438,
//     restricted to base rows because only those enter the ranking, :481-491) and per-column
//     match counts on them (:461-500).
//
//     Bit-parallel: a lane owns one CIGAR op and compares 32 packed bases per step (XOR of 2-bit
//     words).  Per position only the exceptions are counted: coverage and gaps through difference
//     arrays (+-1 at op boundaries, prefix-summed), mismatching bases individually; the count of
//     the target's own allele is coverage - gaps - mismatches + 1.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_pass1(BatchView b) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    const uint32_t W = b.W;
    uint32_t* cnt_ac = (uint32_t*)smem_raw;           // mismatching A | C << 16 per position
    uint32_t* cnt_gt = cnt_ac + W;                    // mismatching G | T << 16
    uint32_t* dcg = cnt_gt + W;                       // [W+1] difference array: coverage (low 16) | gaps (high 16)
    uint64_t* sup2 = (uint64_t*)(dcg + ((W + 2) & ~1u));  // first-pass supported positions, bit 2g of word p/32
    uint64_t* s_t = sup2 + (W >> 5) + 2;              // target window, packed, word-aligned to the window start
    float* key = (float*)(s_t + (W >> 5) + 2);        // MAX_COLS
    uint32_t* cand = (uint32_t*)(key + MAX_COLS);     // MAX_COLS
    __shared__ uint32_t s_n1, s_S, s_warp[8], s_carry;

    const uint32_t w = blockIdx.x;
    const DevWin win = b.win[w];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t n_in = win.ow_end - win.ow_begin;
    if (tid == 0) { s_n1 = 0; s_S = 0; s_carry = 0; }
    __syncthreads();
    if (n_in > MAX_COLS_HARD) {  // the per-position counters are 16 bits wide
        if (tid == 0) { atomicOr(&b.tgt_err[win.tgt], TERR_TOO_MANY_COLS); b.w_n1[w] = 0; b.w_S[w] = 0; }
        return;
    }
    if (n_in > MAX_COLS) {  // the reference has no limit (src/features.rs:376-418): the sort keys of a huge window live in HBM
        key = b.big_key + win.ow_begin;
        cand = b.big_cand + win.ow_begin;
    }
    // ---- filter (order preserving compaction)
    for (uint32_t base = 0; base < n_in; base += 256) {
        const uint32_t i = base + tid;
        const bool keep = i < n_in && !(b.ow_flags[win.ow_begin + i] & (OWF_LONG_INDEL | OWF_BAD));
        const uint32_t m = __ballot_sync(HB_FULL, keep);
        if (lane == 0) s_warp[warp] = __popc(m);
        __syncthreads();
        uint32_t off = s_n1;
        for (int k = 0; k < warp; k++) off += s_warp[k];
        if (keep) {
            const uint32_t pos = off + __popc(m & ((1u << lane) - 1u));
            cand[pos] = win.ow_begin + i;
            key[pos] = -b.ow_acc[win.ow_begin + i];  // OrderedFloat(-acc)
        }
        __syncthreads();
        if (tid == 0) { uint32_t t = 0; for (int k = 0; k < 8; k++) t += s_warp[k]; s_n1 += t; }
        __syncthreads();
    }
    const uint32_t n1 = s_n1;
    // ---- stable ascending sort on key by rank counting
    for (uint32_t i = tid; i < n1; i += 256) {
        const float ki = key[i];
        uint32_t r = 0;
        for (uint32_t j = 0; j < n1; j++) {
            const float kj = key[j];
            r += (kj < ki || (kj == ki && j < i)) ? 1u : 0u;
        }
        b.col_ow[win.ow_begin + r] = cand[i];
    }
    const uint64_t* __restrict__ tw = b.rs.words + b.rs.word_off[win.rid];
    for (uint32_t p = tid; p < W; p += 256) { cnt_ac[p] = 0; cnt_gt[p] = 0; dcg[p] = 0; }
    if (tid == 0) dcg[W] = 0;
    for (uint32_t i = tid; i < (W >> 5) + 2; i += 256) { sup2[i] = 0; s_t[i] = extract32(tw, win.tstart + i * 32); }
    __syncthreads();

    // Both walks are bound by dependent-load latency (column descriptor -> op words -> query words).  Two levels of software
    // pipelining take the first two links off the critical path: the next column's descriptors are fetched while the current
    // column is walked, and a lane's next op words while its current op is compared.
    struct ColCtx { uint32_t owi, op_base, nops, t_first; QView qv; };
    const uint32_t* __restrict__ g_kl = b.op_kl;
    const uint32_t* __restrict__ g_t = b.op_t;
    const uint32_t* __restrict__ g_q = b.op_q;
    auto load_col = [&](uint32_t c) {
        ColCtx x;
        x.owi = cand[c];  // order is irrelevant for counting
        const DevOW ow = b.ow[x.owi];
        x.qv = make_qview(b.rs, b.ovl[ow.ovl], ow);
        x.nops = b.ow_nops[x.owi];
        x.op_base = ow.op_base;
        x.t_first = ow.tstart - win.tstart;
        return x;
    };
    // ---- walk A: coverage / gap difference array and the mismatching bases of every column
    {
        ColCtx nxt{};
        if ((uint32_t)warp < n1) nxt = load_col(warp);
        for (uint32_t c = warp; c < n1; c += 8) {
            const ColCtx cur = nxt;
            if (c + 8 < n1) nxt = load_col(c + 8);
            if (lane == 0) {  // the column covers [p_first, p_end): every position there is an M or a D cell
                atomicAdd(&dcg[cur.t_first], 1u);
                atomicAdd(&dcg[b.ow_tend[cur.owi]], 0xffffffffu);
            }
            uint32_t kl_n = 0, t0_n = 0, q0_n = 0;
            if ((uint32_t)lane < cur.nops) { kl_n = __ldg(g_kl + cur.op_base + lane); t0_n = __ldg(g_t + cur.op_base + lane); q0_n = __ldg(g_q + cur.op_base + lane); }
            for (uint32_t k = lane; k < cur.nops; k += 32) {
                const uint32_t kl = kl_n, t0 = t0_n, q0 = q0_n;
                if (k + 32 < cur.nops) { kl_n = __ldg(g_kl + cur.op_base + k + 32); t0_n = __ldg(g_t + cur.op_base + k + 32); q0_n = __ldg(g_q + cur.op_base + k + 32); }
                const uint32_t kind = kl & 3u, eff = kl >> 2;
                if (kind == OP_I) continue;
                if (kind == OP_D) {
                    atomicAdd(&dcg[t0], 0x10000u);
                    atomicAdd(&dcg[t0 + eff], 0xffff0000u);
                    continue;
                }
                uint64_t qc_next = cur.qv.chunk(q0);
                for (uint32_t i = 0; i < eff; i += 32) {
                    const uint32_t p = t0 + i;
                    // target chunk from the staged window: 32 bases at window-relative position p
                    const uint32_t wi = p >> 5, sh = (p & 31u) << 1;
                    const uint64_t tc = sh ? ((s_t[wi] >> sh) | (s_t[wi + 1] << (64u - sh))) : s_t[wi];
                    const uint64_t qc = qc_next;
                    if (i + 32 < eff) qc_next = cur.qv.chunk(q0 + i + 32);  // next chunk's words in flight while this one's mismatches are counted
                    uint64_t mm = mismatch_groups(tc, qc, eff - i);
                    while (mm) {
                        const int g2 = __ffsll((long long)mm) - 1;  // bit index 2g
                        mm &= mm - 1;
                        const uint32_t cd = (uint32_t)(qc >> g2) & 3u;
                        atomicAdd((cd & 2u) ? &cnt_gt[p + (g2 >> 1)] : &cnt_ac[p + (g2 >> 1)], (cd & 1u) ? 0x10000u : 1u);
                    }
                }
            }
        }
    }
    __syncthreads();
    // ---- prefix-sum the difference array -> coverage | gaps << 16 per position, then the thresholds:
    //      floor(0.1 * ncols) in f64 (src/features.rs:712), >= 2 alleles (:713-718)
    const uint32_t ncols = 1u + (n1 > (uint32_t)TOP_K ? n1 : (uint32_t)TOP_K);
    const uint32_t thresh = (uint32_t)((double)ncols * 0.1);
    uint32_t S_local = 0;
    for (uint32_t base = 0; base < W; base += 256) {
        const uint32_t p = base + tid;
        const uint32_t v = p < win.len ? dcg[p] : 0u;
        const uint32_t inc = warp_incl_scan(v, lane);
        if (lane == 31) s_warp[warp] = inc;
        __syncthreads();
        uint32_t off = s_carry;
        for (int k = 0; k < warp; k++) off += s_warp[k];
        const uint32_t cg = off + inc;  // inclusive: coverage and gaps AT position p
        bool sup = false;
        if (p < win.len) {
            const uint32_t cov = cg & 0xffffu, gp = cg >> 16;
            uint32_t a = cnt_ac[p] & 0xffffu, c = cnt_ac[p] >> 16, g = cnt_gt[p] & 0xffffu, t = cnt_gt[p] >> 16;
            const uint32_t own = cov - gp - (a + c + g + t) + 1u;  // columns agreeing with the target + the target itself
            const uint32_t tc = (uint32_t)(s_t[p >> 5] >> ((p & 31u) << 1)) & 3u;
            a += (tc == 0) ? own : 0; c += (tc == 1) ? own : 0; g += (tc == 2) ? own : 0; t += (tc == 3) ? own : 0;
            const uint32_t ns = (a >= thresh) + (c >= thresh) + (g >= thresh) + (t >= thresh) + (gp >= thresh);
            sup = ns >= 2;
        }
        const uint32_t m = __ballot_sync(HB_FULL, sup);
        if (lane == 0 && m) {
            // spread the 32 flags to the even bits of a 64-bit word (bit 2g <-> position base + 32*warp + g)
            uint64_t x = m;
            x = (x | (x << 16)) & 0x0000ffff0000ffffull;
            x = (x | (x << 8)) & 0x00ff00ff00ff00ffull;
            x = (x | (x << 4)) & 0x0f0f0f0f0f0f0f0full;
            x = (x | (x << 2)) & 0x3333333333333333ull;
            x = (x | (x << 1)) & LOW2;
            sup2[(base >> 5) + warp] = x;
            S_local += __popc(m);
        }
        __syncthreads();
        if (tid == 0) { uint32_t t = 0; for (int k = 0; k < 8; k++) t += s_warp[k]; s_carry += t; }
        __syncthreads();
    }
    if (lane == 0 && S_local) atomicAdd(&s_S, S_local);
    __syncthreads();
    const uint32_t S = s_S;
    // ---- walk B: per-column matches on supported base rows; '.'/gap cells count as mismatches (H1),
    //      hence d = S - n for every column of the window.
    if (S > 0) {
        ColCtx nxt{};
        if ((uint32_t)warp < n1) nxt = load_col(warp);
        for (uint32_t c = warp; c < n1; c += 8) {
            const ColCtx cur = nxt;
            if (c + 8 < n1) nxt = load_col(c + 8);
            uint32_t n = 0;
            uint32_t kl_n = 0, t0_n = 0, q0_n = 0;
            if ((uint32_t)lane < cur.nops) { kl_n = __ldg(g_kl + cur.op_base + lane); t0_n = __ldg(g_t + cur.op_base + lane); q0_n = __ldg(g_q + cur.op_base + lane); }
            for (uint32_t k = lane; k < cur.nops; k += 32) {
                const uint32_t kl = kl_n, t0 = t0_n, q0 = q0_n;
                if (k + 32 < cur.nops) { kl_n = __ldg(g_kl + cur.op_base + k + 32); t0_n = __ldg(g_t + cur.op_base + k + 32); q0_n = __ldg(g_q + cur.op_base + k + 32); }
                if ((kl & 3u) != OP_M) continue;
                const uint32_t eff = kl >> 2;
                for (uint32_t i = 0; i < eff; i += 32) {
                    const uint32_t p = t0 + i;
                    const uint32_t wi = p >> 5, sh = (p & 31u) << 1;
                    const uint64_t sc = sh ? ((sup2[wi] >> sh) | (sup2[wi + 1] << (64u - sh))) : sup2[wi];
                    if (!sc) continue;  // no supported position among these 32: the query words are not even fetched
                    const uint64_t tc = sh ? ((s_t[wi] >> sh) | (s_t[wi + 1] << (64u - sh))) : s_t[wi];
                    const uint64_t mm = mismatch_groups(tc, cur.qv.chunk(q0 + i), eff - i);
                    n += (uint32_t)__popcll(sc & valid_groups(eff - i) & ~mm);
                }
            }
            n = warp_sum(n);
            if (lane == 0) {
                atomicAdd(&b.ovl_n[b.ow[cur.owi].ovl], n);
                atomicAdd(&b.ovl_tot[b.ow[cur.owi].ovl], S);
            }
        }
    }
    if (tid == 0) { b.w_n1[w] = n1; b.w_S[w] = S; }
}

// K3: score = n/(n+d) * ln(n+d+1) in f64 (src/features.rs:505-507); ln from the host-libm table so
//     that it is the value Rust's f64::ln (glibc log) produces.
__global__ void k_scores(BatchView b) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= b.n_ovl) return;
    const uint32_t n = b.ovl_n[i], tot = b.ovl_tot[i];
    double s = 0.0;
    if (tot > 0) {
        const double nd = (double)n, td = (double)tot;
        const uint32_t k = tot + 1u;
        const double l = (k < b.ln_table_n) ? b.ln_table[k] : log((double)k);
        s = __dmul_rn(__ddiv_rn(nd, td), l);
    }
    b.ovl_score[i] = s;
}

// ------------------------------------------------------------------------------------
// K4: second ranking (stable, descending score; src/features.rs:503-513), top-30 selection,
//     max_ins over the selected columns, row map row'(p) and L'.
// ------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_pass2a(BatchView b) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    const uint32_t W = b.W;
    uint32_t* mi = (uint32_t*)smem_raw;            // W + 1
    double* sc = (double*)(mi + ((W + 2) & ~1u));   // MAX_COLS
    if (b.win[blockIdx.x].ow_end - b.win[blockIdx.x].ow_begin > MAX_COLS) sc = b.big_score + b.win[blockIdx.x].ow_begin;
    __shared__ uint32_t s_sel[TOP_K], s_warp[8], s_carry;

    const uint32_t w = blockIdx.x;
    const DevWin win = b.win[w];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t n1 = b.w_n1[w];
    const uint32_t nsel = n1 < (uint32_t)TOP_K ? n1 : (uint32_t)TOP_K;
    for (uint32_t i = tid; i < n1; i += 256) sc[i] = b.ovl_score[b.ow[b.col_ow[win.ow_begin + i]].ovl];
    for (uint32_t p = tid; p <= W; p += 256) mi[p] = 0;
    __syncthreads();
    for (uint32_t i = tid; i < n1; i += 256) {
        const double si = sc[i];
        uint32_t r = 0;
        for (uint32_t j = 0; j < n1; j++) {
            const double sj = sc[j];
            r += (sj > si || (sj == si && j < i)) ? 1u : 0u;
        }
        b.rank_ow[win.ow_begin + r] = b.col_ow[win.ow_begin + i];
        if (r < (uint32_t)TOP_K) {
            s_sel[r] = b.col_ow[win.ow_begin + i];
            b.sel_ow[w * TOP_K + r] = s_sel[r];
        }
    }
    __syncthreads();
    // max_ins over selected columns (src/features.rs:44-95 restricted to the kept columns)
    for (uint32_t c = warp; c < nsel; c += 8) {
        const uint32_t owi = s_sel[c];
        const uint32_t opb = b.ow[owi].op_base, nops = b.ow_nops[owi];
        for (uint32_t k = lane; k < nops; k += 32) {
            const uint32_t kl = b.op_kl[opb + k];
            if ((kl & 3u) == OP_I) {
                const uint32_t tp = b.op_t[opb + k];  // >= 1 (an insertion is never the first op)
                atomicMax(&mi[tp - 1], kl >> 2);
            }
        }
    }
    if (tid == 0) s_carry = 0;
    __syncthreads();
    // exclusive scan of (1 + max_ins[p]) -> row'(p)   (App. A.5)
    uint32_t* rm = b.rowmap + (size_t)w * (W + 1);
    for (uint32_t base = 0; base < win.len; base += 256) {
        const uint32_t p = base + tid;
        const uint32_t v = p < win.len ? 1u + mi[p] : 0u;
        const uint32_t inc = warp_incl_scan(v, lane);
        if (lane == 31) s_warp[warp] = inc;
        __syncthreads();
        uint32_t off = s_carry;
        for (int k = 0; k < warp; k++) off += s_warp[k];
        if (p < win.len) rm[p] = off + inc - v;
        __syncthreads();
        if (tid == 0) { uint32_t t = 0; for (int k = 0; k < 8; k++) t += s_warp[k]; s_carry += t; }
        __syncthreads();
    }
    if (tid == 0) {
        rm[win.len] = s_carry;
        b.w_L[w] = s_carry;
        b.w_nsel[w] = nsel;
    }
}

// K5: exclusive scan of a u32 array into u64 offsets with one block (n up to a few 100k).
__global__ void __launch_bounds__(1024) k_scan_u32(const uint32_t* __restrict__ in, uint64_t* __restrict__ out,
                                                   uint32_t n, uint32_t* counters, int total_slot, uint64_t cap,
                                                   int overflow_slot) {
    __shared__ uint64_t s_warp[32];
    __shared__ uint64_t s_carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < n; base += 1024) {
        const uint32_t i = base + tid;
        const uint64_t v = i < n ? in[i] : 0;
        uint64_t inc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint64_t t = __shfl_up_sync(HB_FULL, inc, o);
            if (lane >= o) inc += t;
        }
        if (lane == 31) s_warp[warp] = inc;
        __syncthreads();
        uint64_t off = s_carry;
        for (int k = 0; k < warp; k++) off += s_warp[k];
        if (i < n) out[i] = off + inc - v;
        __syncthreads();
        if (tid == 0) { uint64_t t = 0; for (int k = 0; k < 32; k++) t += s_warp[k]; s_carry += t; }
        __syncthreads();
    }
    if (tid == 0) {
        counters[total_slot] = (uint32_t)(s_carry & 0xffffffffu);
        counters[total_slot + 1] = (uint32_t)(s_carry >> 32);
        if (overflow_slot >= 0 && s_carry > cap) counters[overflow_slot] = 1;
    }
}

// ------------------------------------------------------------------------------------
// K7: build the final [L',31] token/quality matrix of one window tile by tile in shared
//     memory, evaluate the second get_supported (thresh = floor(3.1) = 3) and the majority vote
//     on the tile, and stream the tile to HBM with 16-byte stores.          (the pileup kernel)
// ------------------------------------------------------------------------------------
constexpr int TR = 512;      // rows per tile
constexpr int QSTAGE = 1024;  // staged quality bytes per warp (>= TR + a straddling op)
constexpr int OPCAP = 96;     // staged ops per warp and column-tile (falls back to global memory beyond)

__global__ void __launch_bounds__(256) k_pass2b(BatchView b) {
    // tile in shared memory, column-major ("planes"): plane c holds the TR tokens / quals of column c, so a column's
    // consecutive rows are consecutive bytes (conflict-free scatter); rows are gathered per thread for the row-wise
    // work and written to HBM row-major ([L',32], 32-byte rows).
    extern __shared__ __align__(16) uint8_t smem_raw[];
    uint8_t* p_tok = smem_raw;                    // [32][TR]
    uint8_t* p_q = p_tok + 32 * TR;               // [32][TR]
    uint32_t* rm_s = (uint32_t*)(p_q + 32 * TR);  // [TR + 2]
    uint32_t* pk_s = rm_s + TR + 2;               // [TR]
    uint8_t* sup_s = (uint8_t*)(pk_s + TR);       // [TR]
    uint8_t* q_stage = sup_s + TR;                // [8 warps][QSTAGE] staged quality bytes of the column being expanded
    uint32_t* op_stage = (uint32_t*)(q_stage + 8 * QSTAGE);  // [8 warps][3][OPCAP] staged ops of the column-tile
    __shared__ uint32_t c_ow[32], c_rs[32], c_re[32], c_gap[32];
    __shared__ uint32_t s_phi, s_warp[8], s_nsup;
    __shared__ uint32_t s_khint[8][4];  // per (warp, column slot): where the previous tile's op search ended

    const uint32_t w = blockIdx.x;
    const DevWin win = b.win[w];
    const uint32_t W = b.W;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t nsel = b.w_nsel[w];
    const uint32_t L = b.w_L[w];
    const uint64_t rowbase = b.w_rowbase[w];
    if (b.counters[CNT_OVERFLOW]) return;  // arena too small: host grows it and re-launches
    const uint32_t* __restrict__ rm = b.rowmap + (size_t)w * (W + 1);
    const uint64_t* __restrict__ tw = b.rs.words + b.rs.word_off[win.rid];
    const uint8_t* __restrict__ tq = b.rs.qual + b.rs.qual_off[win.rid] + win.tstart;

    if (tid < 32) {
        uint32_t owi = 0, rs = 0, re = 0, gap = TOK_NONE;
        if (tid >= 1 && (uint32_t)tid <= nsel) {
            owi = b.sel_ow[w * TOP_K + tid - 1];
            const DevOW ow = b.ow[owi];
            rs = rm[ow.tstart - win.tstart];       // rows before are '.' (src/features.rs:166-171)
            re = rm[b.ow_tend[owi]];               // rows from here on are '.' (:233-236)
            gap = b.ovl[ow.ovl].strand ? TOK_GAP_R : TOK_GAP_F;
        } else if (tid == 0) {
            rs = 0; re = L; gap = TOK_GAP_F;       // target column: bases.fill('*') (:248)
        }
        c_ow[tid] = owi; c_rs[tid] = rs; c_re[tid] = re; c_gap[tid] = gap;
    }
    if (tid == 0) s_nsup = 0;
    if (tid < 32) s_khint[tid >> 2][tid & 3] = 0;

    uint32_t p_lo = 0;
    __syncthreads();

    for (uint32_t r0 = 0; r0 < L; r0 += TR) {
        const uint32_t r1 = min(r0 + (uint32_t)TR, L);
        // ---- positions touching this tile: p_lo .. p_hi-1 ; rm_s[i] = row'(p_lo + i)
        for (uint32_t i = tid; i < TR + 2; i += 256) {
            const uint32_t p = p_lo + i;
            rm_s[i] = p <= win.len ? rm[p] : 0xffffffffu;
        }
        __syncthreads();
        for (uint32_t i = tid; i < TR + 1; i += 256) {
            // first p with row'(p) >= r1
            if (rm_s[i] >= r1 && (i == 0 || rm_s[i - 1] < r1)) s_phi = p_lo + i;
        }
        // ---- initial fill per plane, 16 rows per store: gap inside the column's aligned row range, '.' outside, '!' quals
        for (uint32_t i = tid; i < 32u * (TR / 16); i += 256) {
            const uint32_t c = i / (TR / 16), seg = i % (TR / 16);
            const uint32_t row0 = r0 + seg * 16;
            const uint32_t rs = c_rs[c], re = c_re[c], gap = c_gap[c];
            uint32_t wv[4];
            if (row0 >= rs && row0 + 16 <= re) {
                wv[0] = wv[1] = wv[2] = wv[3] = gap * 0x01010101u;
            } else if (row0 + 16 <= rs || row0 >= re) {
                wv[0] = wv[1] = wv[2] = wv[3] = TOK_NONE * 0x01010101u;
            } else {
#pragma unroll
                for (int q4 = 0; q4 < 4; q4++) {
                    uint32_t x = 0;
#pragma unroll
                    for (int e = 0; e < 4; e++) {
                        const uint32_t row = row0 + q4 * 4 + e;
                        x |= ((row >= rs && row < re) ? gap : TOK_NONE) << (8 * e);
                    }
                    wv[q4] = x;
                }
            }
            *(uint4*)(p_tok + c * TR + seg * 16) = make_uint4(wv[0], wv[1], wv[2], wv[3]);
            *(uint4*)(p_q + c * TR + seg * 16) = make_uint4(0x21212121u, 0x21212121u, 0x21212121u, 0x21212121u);
        }
        __syncthreads();
        const uint32_t p_hi = s_phi;
        // ---- target column + (pos, ins) of every row
        for (uint32_t p = p_lo + tid; p < p_hi; p += 256) {
            const uint32_t row = rm_s[p - p_lo], nxt = rm_s[p - p_lo + 1];
            if (row >= r0) {
                p_tok[row - r0] = (uint8_t)code_at(tw, win.tstart + p);
                p_q[row - r0] = __ldg(tq + p);
            }
            for (uint32_t k = 0; row + k < nxt; k++) {
                const uint32_t r = row + k;
                if (r >= r0 && r < r1) pk_s[r - r0] = (p << 8) | (k & 0xffu);
            }
        }
        // ---- overlap columns.  A warp owns a column; each lane owns an equal slice of the tile's target positions,
        //      finds the op covering its first position by binary search and walks forward, expanding the packed query
        //      bases (32 per 64-bit word) into the plane.  The column's quality bytes for the tile are staged through a
        //      per-warp buffer with coalesced loads first (the L1 of this kernel is mostly carved out as shared memory).
        {
            const uint32_t npos = p_hi - p_lo;
            const uint32_t seg = (npos + 31) / 32;
            const uint32_t a = p_lo + lane * seg, bnd = min(p_hi, a + seg);  // this lane's positions [a, bnd)
            uint8_t* qst = q_stage + warp * QSTAGE;
#pragma unroll 1
            for (int s_ = 0; s_ < 4; s_++) {
                const uint32_t c = 1 + warp + 8 * s_;
                if (c > nsel) break;
                const uint32_t owi = c_ow[c];
                const DevOW ow = b.ow[owi];
                const QView qv = make_qview(b.rs, b.ovl[ow.ovl], ow);
                uint32_t nops = b.ow_nops[owi];
                const uint32_t* okl = b.op_kl + ow.op_base;
                const uint32_t* opt = b.op_t + ow.op_base;
                const uint32_t* opq = b.op_q + ow.op_base;
                const uint32_t add = qv.rev ? 5u : 0u;
                uint8_t* pt = p_tok + c * TR;
                uint8_t* pq = p_q + c * TR;
                // first op with op_t >= p_lo.  op_t is sorted and p_lo grows from tile to tile, so the search resumes at the
                // previous tile's answer for this column and probes 32 ops per step (one coalesced load, one ballot): the
                // former warp-uniform binary searches were ~7 dependent global loads each, 13 % of the kernel's stall samples.
                uint32_t lo_k;
                for (uint32_t base = s_khint[warp][s_];; base += 32) {  // invariant: every op before `base` has op_t < p_lo
                    const uint32_t idx = base + lane;
                    const uint32_t m = __ballot_sync(HB_FULL, idx >= nops || opt[idx] >= p_lo);
                    if (m) { lo_k = min(base + (uint32_t)__ffs(m) - 1u, nops); break; }
                }
                uint32_t k_first = lo_k;  // first op with op_t >= p_lo ...
                if (k_first > 0) k_first--;  // ... and the one before it, which may straddle p_lo
                if (lane == 0) s_khint[warp][s_] = k_first;
                const uint32_t qbase = k_first < nops ? opq[k_first] : 0;  // oriented offset where the staged window starts
                const uint32_t qslice = ow.qend - ow.qstart;
                // ... and where it ends: the query offset of the first op that starts after the tile's positions
                uint32_t lo_e;  // first op in [k_first, nops) with op_t > p_hi, same probing
                for (uint32_t base = k_first;; base += 32) {
                    const uint32_t idx = base + lane;
                    const uint32_t m = __ballot_sync(HB_FULL, idx >= nops || opt[idx] > p_hi);
                    if (m) { lo_e = min(base + (uint32_t)__ffs(m) - 1u, nops); break; }
                }
                const uint32_t qend_t = lo_e < nops ? opq[lo_e] : qslice;
                const uint32_t qn = min((uint32_t)QSTAGE, qend_t > qbase ? qend_t - qbase : 0u);
                const uint32_t qn4 = qn >> 2;                      // whole 4-byte words of the staged window
                for (uint32_t w0 = 0; w0 < qn4; w0 += 128) {       // 4 independent word fetches in flight per lane
                    uint32_t v[4];
#pragma unroll
                    for (int u = 0; u < 4; u++) { const uint32_t wi = w0 + u * 32 + lane; v[u] = wi < qn4 ? qv.q4(qbase + 4 * wi) : 0; }
#pragma unroll
                    for (int u = 0; u < 4; u++) { const uint32_t wi = w0 + u * 32 + lane; if (wi < qn4) ((uint32_t*)qst)[wi] = v[u]; }
                }
                for (uint32_t i = 4 * qn4 + lane; i < qn; i += 32) qst[i] = qv.q(qbase + i);  // the last 0..3 bytes
                // stage the ops that touch this tile (k_first .. lo_e) so that the lanes' searches and walks read shared memory
                const uint32_t ne = min(nops, lo_e + 1) - k_first;
                if (ne <= (uint32_t)OPCAP) {
                    uint32_t* so = op_stage + warp * 3 * OPCAP;
                    for (uint32_t i = lane; i < ne; i += 32) {
                        so[i] = okl[k_first + i]; so[OPCAP + i] = opt[k_first + i]; so[2 * OPCAP + i] = opq[k_first + i];
                    }
                    okl = so - k_first; opt = so + OPCAP - k_first; opq = so + 2 * OPCAP - k_first;  // keep global op indices
                    nops = k_first + ne;
                }
                __syncwarp();
                if (a < bnd) {
                    // lane-local search: first op with op_t >= a, then step back to a straddling M/D op
                    uint32_t l2 = k_first, h2 = nops;
                    while (l2 < h2) {
                        const uint32_t mid = (l2 + h2) >> 1;
                        if (opt[mid] < a) l2 = mid + 1; else h2 = mid;
                    }
                    uint32_t k = l2;
                    if (k > 0) {
                        const uint32_t klp = okl[k - 1];
                        if ((klp & 3u) != OP_I && opt[k - 1] + (klp >> 2) > a) k--;
                    }
                    // flat walk over this lane's positions: every lane runs the same ~seg iterations
                    uint32_t kind = OP_D, op_end = a, xq = 0;  // current op: covers positions [.., op_end), next query offset xq
                    uint64_t qc = 0;
                    uint32_t cbase = 0;                        // query offset of qc's first base
                    bool have_qc = false;
                    for (uint32_t p = a; p < bnd; p++) {
                        while (p >= op_end && k < nops) {      // advance to the op covering p, expanding insertions on the way
                            const uint32_t kl = okl[k];
                            const uint32_t kd = kl & 3u, eff = kl >> 2, t0 = opt[k];
                            if (kd == OP_I) {
                                const uint32_t pp = t0 - 1;    // insertion after position pp; ours iff a <= pp (pp < p holds here)
                                if (pp >= a && pp < bnd) {
                                    const uint32_t q0 = opq[k], rb = rm_s[pp - p_lo] + 1;
                                    for (uint32_t j = 0; j < eff; j++) {
                                        const uint32_t r = rb + j;
                                        if (r >= r0 && r < r1) {
                                            pt[r - r0] = (uint8_t)(qv.code(q0 + j) + add);
                                            const uint32_t x = q0 + j;
                                            pq[r - r0] = (x - qbase < qn) ? qst[x - qbase] : qv.q(x);
                                        }
                                    }
                                }
                                k++;
                                continue;
                            }
                            if (t0 > p) { kind = OP_D; op_end = t0; break; }  // uncovered gap before the next op (cannot happen inside an overlap)
                            kind = kd; op_end = t0 + eff; xq = opq[k] + (p - t0);
                            k++;
                        }
                        if (p >= op_end) break;                // past the column's last op
                        if (kind == OP_M) {
                            if (!have_qc || xq - cbase >= 32u) { cbase = xq; qc = qv.chunk(cbase); have_qc = true; }
                            const uint32_t r = rm_s[p - p_lo];
                            if (r >= r0) {
                                pt[r - r0] = (uint8_t)(((uint32_t)(qc >> (2u * (xq - cbase))) & 3u) + add);
                                pq[r - r0] = (xq - qbase < qn) ? qst[xq - qbase] : qv.q(xq);
                            }
                            xq++;
                        }
                    }
                    // an insertion right after this lane's last position (op_t == bnd) belongs to this lane
                    while (k < nops && opt[k] <= bnd) {
                        const uint32_t kl = okl[k];
                        if ((kl & 3u) == OP_I && opt[k] == bnd && bnd - 1 >= a) {
                            const uint32_t eff = kl >> 2, q0 = opq[k], rb = rm_s[bnd - 1 - p_lo] + 1;
                            for (uint32_t j = 0; j < eff; j++) {
                                const uint32_t r = rb + j;
                                if (r >= r0 && r < r1) {
                                    pt[r - r0] = (uint8_t)(qv.code(q0 + j) + add);
                                    const uint32_t x = q0 + j;
                                    pq[r - r0] = (x - qbase < qn) ? qst[x - qbase] : qv.q(x);
                                }
                            }
                        }
                        if ((kl & 3u) != OP_I) break;
                        k++;
                    }
                }
                __syncwarp();  // the staging buffer is reused by the next column
            }
        }
        __syncthreads();
        // ---- per-row work, one thread per row: gather the row from the planes, second get_supported
        //      (src/features.rs:681-722 on [L',31], thresh 3) and the majority vote of consensus
        //      (src/consensus.rs:176-200) with byte-parallel class counts, row-major 32-byte stores to HBM.
        for (uint32_t rr = tid; rr < r1 - r0; rr += 256) {
            uint32_t wv[8], qw[8];
#pragma unroll
            for (int i = 0; i < 8; i++) {
                uint32_t x = 0, y = 0;
#pragma unroll
                for (int e = 0; e < 4; e++) {
                    x |= (uint32_t)p_tok[(i * 4 + e) * TR + rr] << (8 * e);
                    y |= (uint32_t)p_q[(i * 4 + e) * TR + rr] << (8 * e);
                }
                wv[i] = x; qw[i] = y;
            }
            uint32_t cnt[5] = {0, 0, 0, 0, 0};
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const uint32_t x = wv[i];
                const uint32_t cls = __vsub4(x, __vcmpgeu4(x, 0x05050505u) & 0x05050505u);  // BASES_UPPER_COUNTER / BASE_FORWARD
                const uint32_t live = __vcmpltu4(x, 0x0a0a0a0au);                            // token < '.'
#pragma unroll
                for (int k = 0; k < 5; k++) cnt[k] += __popc(__vcmpeq4(cls, 0x01010101u * (uint32_t)k) & live & 0x01010101u);
            }
            const uint32_t ns = (cnt[0] >= 3) + (cnt[1] >= 3) + (cnt[2] >= 3) + (cnt[3] >= 3) + (cnt[4] >= 3);
            const bool sup = ns >= 2;
            // two most common, stable on ties (A<C<G<T<*)
            uint32_t b0 = 0;
#pragma unroll
            for (int k = 1; k < 5; k++) if (cnt[k] > cnt[b0]) b0 = k;
            uint32_t b1 = b0 == 0 ? 1 : 0;
#pragma unroll
            for (int k = 0; k < 5; k++) if ((uint32_t)k != b0 && (uint32_t)k != b1 && cnt[k] > cnt[b1]) b1 = k;
            const uint32_t tb = wv[0] & 0xffu;  // target column, token 0..4
            const uint32_t base = (cnt[b0] < 2 || (cnt[b0] == cnt[b1] && (b0 == tb || b1 == tb))) ? tb : b0;
            const uint32_t emit = nsel >= 2 ? base : 4u;  // n_alns < 2: window dropped (src/consensus.rs:104-111)
            b.row_emit[rowbase + r0 + rr] = (uint8_t)(emit | (sup ? 0x80u : 0u));
            sup_s[rr] = sup ? 1 : 0;
            uint4* gb = (uint4*)(b.mat_bases + (rowbase + r0 + rr) * ROW_BYTES);
            uint4* gq = (uint4*)(b.mat_quals + (rowbase + r0 + rr) * ROW_BYTES);
            gb[0] = make_uint4(wv[0], wv[1], wv[2], wv[3]); gb[1] = make_uint4(wv[4], wv[5], wv[6], wv[7]);
            gq[0] = make_uint4(qw[0], qw[1], qw[2], qw[3]); gq[1] = make_uint4(qw[4], qw[5], qw[6], qw[7]);
        }
        __syncthreads();
        // ---- ordered list of supported rows
        for (uint32_t base = 0; base < r1 - r0; base += 256) {
            const uint32_t rr = base + tid;
            const bool f = rr < r1 - r0 && sup_s[rr];
            const uint32_t m = __ballot_sync(HB_FULL, f);
            if (lane == 0) s_warp[warp] = __popc(m);
            __syncthreads();
            uint32_t off = s_nsup;
            for (int k = 0; k < warp; k++) off += s_warp[k];
            if (f) {
                const uint32_t pos = off + __popc(m & ((1u << lane) - 1u));
                b.sup_row[rowbase + pos] = r0 + rr;
                b.sup_pk[rowbase + pos] = pk_s[rr];
            }
            __syncthreads();
            if (tid == 0) { uint32_t t = 0; for (int k = 0; k < 8; k++) t += s_warp[k]; s_nsup += t; }
            __syncthreads();
        }
        // next tile starts at the position whose rows straddle r1
        p_lo = (p_hi <= win.len && p_hi > 0 && rm_s[p_hi - p_lo] == r1) ? p_hi : p_hi - 1;
        __syncthreads();
    }
    if (tid == 0) b.w_nsup[w] = s_nsup;
}

// K6: Lmax of the reference's collate batch (src/inference.rs:73-84) for each window: the
//     reference flushes after `-b` consecutive windows of a read and at the end of the read
//     (src/features.rs:884-893); the windows with >= 1 supported row of such a group form one
//     batch tensor padded to the longest of them.
__global__ void k_ref_lmax(BatchView b) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= b.n_tgt) return;
    const DevTarget tg = b.tgt[t];
    for (uint32_t g0 = tg.win_begin; g0 < tg.win_end; g0 += b.batch_size) {
        const uint32_t g1 = min(g0 + b.batch_size, tg.win_end);
        uint32_t lmax = 0;
        for (uint32_t w = g0; w < g1; w++) if (b.w_nsup[w] > 0) lmax = max(lmax, b.w_L[w]);
        for (uint32_t w = g0; w < g1; w++) b.w_reflmax[w] = lmax;
    }
}

// K8: flatten the per-window supported lists into the forward work list.
__global__ void __launch_bounds__(256) k_fwd_list(BatchView b) {
    const uint32_t w = blockIdx.x;
    const uint32_t n = b.w_nsup[w];
    const uint64_t src = b.w_rowbase[w], dst = b.w_supbase[w];
    for (uint32_t i = threadIdx.x; i < n; i += 256) {
        b.fwd_win[dst + i] = w;
        b.fwd_row[dst + i] = b.sup_row[src + i];
    }
}

// ------------------------------------------------------------------------------------
// Consensus: count / write the emitted bases of every window (src/consensus.rs:103-224).
// row_emit already holds the majority-vote base of every row and, for supported rows, the
// argmax class written by the forward head (H9).
// ------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_cons_count(BatchView b) {
    __shared__ uint32_t s_tot;
    const uint32_t w = blockIdx.x;
    if (threadIdx.x == 0) s_tot = 0;
    __syncthreads();
    const uint32_t L = b.w_L[w];
    const uint8_t* e = b.row_emit + b.w_rowbase[w];
    uint32_t c = 0;
    if (b.w_nsel[w] >= 2)
        for (uint32_t r = threadIdx.x; r < L; r += 256) c += ((e[r] & 7u) != 4u) ? 1u : 0u;
    c = warp_sum(c);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(&s_tot, c);
    __syncthreads();
    if (threadIdx.x == 0) b.w_outlen[w] = s_tot;
}

__global__ void __launch_bounds__(256) k_cons_write(BatchView b) {
    __shared__ uint32_t s_warp[8], s_carry;
    const uint32_t w = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (b.w_outlen[w] == 0) return;
    const uint32_t L = b.w_L[w];
    const uint8_t* e = b.row_emit + b.w_rowbase[w];
    uint8_t* out = b.out_bytes + b.w_outoff[w];
    if (tid == 0) s_carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < L; base += 256) {
        const uint32_t r = base + tid;
        const uint32_t cls = r < L ? (e[r] & 7u) : 4u;
        const bool f = cls != 4u;
        const uint32_t m = __ballot_sync(HB_FULL, f);
        if (lane == 0) s_warp[warp] = __popc(m);
        __syncthreads();
        uint32_t off = s_carry;
        for (int k = 0; k < warp; k++) off += s_warp[k];
        if (f) out[off + __popc(m & ((1u << lane) - 1u))] = "ACGT"[cls];
        __syncthreads();
        if (tid == 0) { uint32_t t = 0; for (int k = 0; k < 8; k++) t += s_warp[k]; s_carry += t; }
        __syncthreads();
    }
}

void launch_scan_u32(const uint32_t* in, uint64_t* out, uint32_t n, uint32_t* counters, int total_slot, uint64_t cap, int overflow_slot,
                     cudaStream_t st) {
    k_scan_u32<<<1, 1024, 0, st>>>(in, out, n, counters, total_slot, cap, overflow_slot);
}

// ------------------------------------------------------------------------------------
// launch wrappers (called from ctx.cu)
// ------------------------------------------------------------------------------------
size_t pass1_smem(uint32_t W) { return (size_t)W * 8 + (size_t)((W + 2) & ~1u) * 4 + 2 * ((W >> 5) + 2) * 8 + MAX_COLS * 8 + 64; }
size_t pass2b_smem() { return (size_t)64 * TR + (TR + 2) * 4 + TR * 4 + TR + 8 * QSTAGE + 8 * 3 * OPCAP * 4 + 64; }
size_t pass2a_smem(uint32_t W) { return (size_t)((W + 2) & ~1u) * 4 + MAX_COLS * 8 + 64; }

cudaError_t features_configure(uint32_t W) {
    cudaError_t e = cudaFuncSetAttribute(k_pass1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pass1_smem(W));
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(k_pass2a, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pass2a_smem(W));
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(k_pass2b, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pass2b_smem());
    if (e != cudaSuccess) return e;
    return pileup_configure();
}

int launch_features_a(const BatchView& b, cudaStream_t st, KTimer& kt) {
    int n = 0;
    if (b.n_ow) {
        kt.begin(K_TOKENIZE);
        if (b.n_raw) n += launch_windowing(b, st);  // device extract_windows for the alignments submitted raw
        if (b.n_raw) { k_tokenize<true><<<(b.n_ow * 32 + 127) / 128, 128, 0, st>>>(b); n++; }
        if (b.n_raw < b.n_ovl) { k_tokenize<false><<<(b.n_ow * 32 + 127) / 128, 128, 0, st>>>(b); n++; }
        kt.end();
    }
    kt.begin(K_PASS1); k_pass1<<<b.n_win, 256, pass1_smem(b.W), st>>>(b); kt.end(); n++;
    if (b.n_ovl) { kt.begin(K_SCORES); k_scores<<<(b.n_ovl + 255) / 256, 256, 0, st>>>(b); kt.end(); n++; }
    kt.begin(K_PASS2A); k_pass2a<<<b.n_win, 256, pass2a_smem(b.W), st>>>(b); kt.end(); n++;
    kt.begin(K_SCAN);
    k_scan_u32<<<1, 1024, 0, st>>>(b.w_L, b.w_rowbase, b.n_win, b.counters, CNT_TOTAL_ROWS, b.rows_cap, CNT_OVERFLOW);
    kt.end(); n++;
    return n;
}
int launch_pileup(const BatchView& b, cudaStream_t st, KTimer& kt, bool v1) {
    kt.begin(K_PILEUP);
    if (v1) k_pass2b<<<b.n_win, 256, pass2b_smem(), st>>>(b);  // former position-walk kernel (A-B parity test only)
    else launch_pileup_v2(b, st);
    kt.end();
    return 1;
}
int launch_features_c1(const BatchView& b, cudaStream_t st, KTimer& kt) {
    kt.begin(K_LISTS); k_ref_lmax<<<(b.n_tgt + 127) / 128, 128, 0, st>>>(b); kt.end();
    kt.begin(K_SCAN); k_scan_u32<<<1, 1024, 0, st>>>(b.w_nsup, b.w_supbase, b.n_win, b.counters, CNT_NSUP, 0, -1); kt.end();
    return 2;
}
int launch_features_c2(const BatchView& b, cudaStream_t st, KTimer& kt) {
    kt.begin(K_LISTS); k_fwd_list<<<b.n_win, 256, 0, st>>>(b); kt.end();
    return 1;
}
int launch_consensus(const BatchView& b, cudaStream_t st, KTimer& kt) {
    kt.begin(K_CONSENSUS); k_cons_count<<<b.n_win, 256, 0, st>>>(b); kt.end();
    kt.begin(K_SCAN); k_scan_u32<<<1, 1024, 0, st>>>(b.w_outlen, b.w_outoff, b.n_win, b.counters, CNT_TOTAL_OUT, 0, -1); kt.end();
    kt.begin(K_CONSENSUS); k_cons_write<<<b.n_win, 256, 0, st>>>(b); kt.end();
    return 3;
}

}  // namespace hb
