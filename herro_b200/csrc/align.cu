// align.cu — the base-level alignment of overlaps (hb_align_overlaps, DESIGN.md §12): a banded two-piece Gotoh over the target
// slice and the oriented query slice of every overlap, its traceback, fix_cigar, the end-gap trim and the CIGAR text.
//
// k_align_fill: one warp per overlap, rows (target positions) in order.  Lane l owns the P consecutive cells [lP, lP + P) of the
// row's band (2w cells, P = 2w / 32 rounded up to a power of two; cells past 2w are outside the band).  The previous row's H, F1
// and F2 stay in registers and are shifted by the band's move c(i) - c(i-1) (0..2 cells) with shuffles.  The horizontal states
// are resolved inside the row by a warp max-scan of H'(k) + e k per gap piece, H' being H without E: exact, since two adjacent
// gaps always cost more than one gap of their total length (DESIGN.md §12.2).  Each row's traceback bytes (bits 0-2: H's source
// 0 diag, 1 F1, 2 F2, 3 E1, 4 E2; bits 3-6: F1, F2, E1, E2 extended) leave as one coalesced store of 2w bytes.
// k_align_trace: one thread per overlap walks back from (n, m), run-length encodes, applies fix_cigar, trims end gaps, counts the
// identical pairs inside M and the CIGAR's text length.  k_align_text writes the text at offsets the host scanned.
#include "common.cuh"
#include "forward.h"

namespace hb {

namespace {

constexpr int32_t A_NEG = -(1 << 30);  // outside the band; every state is clamped to it, so nothing can overflow
constexpr int AF_WARPS = 4;
constexpr int AT_THREADS = 128;
constexpr uint32_t A_M = 0, A_I = 1, A_D = 2;

__device__ __forceinline__ int32_t cl(int32_t v) { return max(v, A_NEG); }

// o[t] = a at row cell lane * P + t + S (A_NEG outside the warp's cells); S is a compile-time shift, so every index is too
template <int P, int S>
__device__ __forceinline__ void shift_cells(const int32_t (&a)[P], int32_t (&o)[P], int lane) {
#pragma unroll
    for (int t = 0; t < P; t++) {
        const int x = t + S;
        const int dl = x >= 0 ? x / P : -((P - 1 - x) / P);
        const int e = x - dl * P;
        int32_t v = a[e];
        if (dl != 0) {
            v = __shfl_sync(HB_FULL, v, (lane + dl) & 31);
            if (lane + dl < 0 || lane + dl > 31) v = A_NEG;
        }
        o[t] = v;
    }
}

template <int P>
__device__ __forceinline__ void shift_rt(const int32_t (&a)[P], int32_t (&o)[P], int lane, int s) {
    switch (s) {
        case -1: shift_cells<P, -1>(a, o, lane); break;
        case 0: shift_cells<P, 0>(a, o, lane); break;
        case 1: shift_cells<P, 1>(a, o, lane); break;
        default: shift_cells<P, 2>(a, o, lane); break;
    }
}

template <int P> struct RowVec;
template <> struct RowVec<1> { using T = uint8_t; };
template <> struct RowVec<2> { using T = uint16_t; };
template <> struct RowVec<4> { using T = uint32_t; };
template <> struct RowVec<8> { using T = uint2; };
template <> struct RowVec<16> { using T = uint4; };

template <int P>
__device__ __forceinline__ void store_row(uint8_t* dst, const uint32_t (&b)[P]) {
    typename RowVec<P>::T v;
    uint32_t* u = (uint32_t*)&v;
    if constexpr (P == 1) {
        v = (uint8_t)b[0];
    } else if constexpr (P == 2) {
        v = (uint16_t)(b[0] | b[1] << 8);
    } else {
#pragma unroll
        for (int k = 0; k < P / 4; k++) u[k] = b[4 * k] | b[4 * k + 1] << 8 | b[4 * k + 2] << 16 | b[4 * k + 3] << 24;
    }
    *(typename RowVec<P>::T*)dst = v;
}

__device__ __forceinline__ QView job_qview(const ReadStoreView& rs, const AlnJob& J) {
    QView v;
    v.words = rs.words + rs.word_off[J.qid];
    v.qual = nullptr;
    v.qs = J.qstart;
    v.qe = J.qend;
    v.rev = J.strand;
    return v;
}

template <int P>
__global__ void __launch_bounds__(AF_WARPS * 32) k_align_fill(AlnArgs a) {
    const uint32_t jid = blockIdx.x * AF_WARPS + (threadIdx.x >> 5);
    if (jid >= a.n_jobs) return;
    const int lane = threadIdx.x & 31;
    const AlnJob J = a.jobs[jid];
    const int32_t w = (int32_t)a.w, W2 = 2 * w;
    const uint32_t n = J.tend - J.tstart, m = J.qend - J.qstart;
    const uint64_t* tw = a.rs.words + a.rs.word_off[J.tid];
    const QView qv = job_qview(a.rs, J);
    uint8_t* tb = a.tb + J.tb_off;
    int32_t pH[P], pF1[P], pF2[P];
#pragma unroll
    for (int t = 0; t < P; t++) pH[t] = pF1[t] = pF2[t] = A_NEG;
    uint32_t cprev = 0;
    for (uint32_t i = 0; i <= n; i++) {
        const uint32_t ci = (uint32_t)(((uint64_t)i * m) / n);
        const int d = (int)(ci - cprev);
        cprev = ci;
        const int64_t j0 = (int64_t)ci - w + lane * P;  // column of the lane's first cell
        int32_t x[P], y[P];
        uint32_t bits[P];
        // vertical states from the cells above (shift d)
        shift_rt<P>(pH, x, lane, d);
        shift_rt<P>(pF1, y, lane, d);
#pragma unroll
        for (int t = 0; t < P; t++) {
            const int32_t o = cl(x[t] - 6), e = cl(y[t] - 2);
            bits[t] = (e >= o) << 3;
            pF1[t] = max(o, e);
        }
        shift_rt<P>(pF2, y, lane, d);
#pragma unroll
        for (int t = 0; t < P; t++) {
            const int32_t o = cl(x[t] - 25), e = cl(y[t] - 1);
            bits[t] |= (e >= o) << 4;
            pF2[t] = max(o, e);
        }
        // diagonal (shift d - 1); the row's target base and the lane's query bases j - 1 from one 32-base chunk
        shift_rt<P>(pH, x, lane, d - 1);
        const uint32_t tbase = i ? code_at(tw, J.tstart + i - 1) : 0u;
        const int64_t x0 = j0 - 1 < 0 ? 0 : j0 - 1;
        const uint64_t qc = x0 < (int64_t)m ? qv.chunk((uint32_t)x0) : 0ull;
#pragma unroll
        for (int t = 0; t < P; t++) {
            const int64_t j = j0 + t;
            const bool valid = lane * P + t < W2 && j >= 0 && j <= (int64_t)m;
            int32_t h = A_NEG;
            uint32_t src = 0;
            if (i > 0 && j > 0) {
                const uint32_t qb = (uint32_t)(qc >> (2 * (j - 1 - x0))) & 3u;
                h = cl(x[t] + (qb == tbase ? 2 : -4));
            }
            if (pF1[t] > h) { h = pF1[t]; src = 1; }
            if (pF2[t] > h) { h = pF2[t]; src = 2; }
            if (i == 0 && j == 0) h = 0;
            if (!valid) { h = A_NEG; pF1[t] = A_NEG; pF2[t] = A_NEG; }
            pH[t] = h;  // H' for now
            bits[t] |= src;
        }
        // horizontal states: E(k) = max_{k' < k} H'(k') - q - e (k - k'), by an exclusive max-scan of H'(k') + e k' per piece
        int32_t e1[P], e2[P];
        {
            int32_t r1 = A_NEG, r2 = A_NEG;
#pragma unroll
            for (int t = 0; t < P; t++) {
                const int32_t k = lane * P + t;
                e1[t] = r1;
                e2[t] = r2;
                r1 = max(r1, pH[t] + 2 * k);
                r2 = max(r2, pH[t] + k);
            }
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int32_t v1 = __shfl_up_sync(HB_FULL, r1, o), v2 = __shfl_up_sync(HB_FULL, r2, o);
                if (lane >= o) { r1 = max(r1, v1); r2 = max(r2, v2); }
            }
            int32_t x1 = __shfl_up_sync(HB_FULL, r1, 1), x2 = __shfl_up_sync(HB_FULL, r2, 1);
            if (lane == 0) x1 = x2 = A_NEG;
#pragma unroll
            for (int t = 0; t < P; t++) {
                const int32_t k = lane * P + t;
                e1[t] = cl(max(x1, e1[t]) - 4 - 2 * k);
                e2[t] = cl(max(x2, e2[t]) - 24 - k);
            }
        }
#pragma unroll
        for (int t = 0; t < P; t++) {
            const int64_t j = j0 + t;
            const bool valid = lane * P + t < W2 && j >= 0 && j <= (int64_t)m;
            int32_t h = pH[t];
            if (e1[t] > h) { h = e1[t]; bits[t] = (bits[t] & ~7u) | 3u; }
            if (e2[t] > h) { h = e2[t]; bits[t] = (bits[t] & ~7u) | 4u; }
            pH[t] = valid ? h : A_NEG;
        }
        // extension bits of the horizontal states, from the left neighbour's E and H
        shift_cells<P, -1>(pH, x, lane);
        shift_cells<P, -1>(e1, y, lane);
#pragma unroll
        for (int t = 0; t < P; t++) bits[t] |= (cl(y[t] - 2) >= cl(x[t] - 6)) << 5;
        shift_cells<P, -1>(e2, y, lane);
#pragma unroll
        for (int t = 0; t < P; t++) bits[t] |= (cl(y[t] - 1) >= cl(x[t] - 25)) << 6;
        if (lane * P < W2) store_row<P>(tb + (uint64_t)i * W2 + lane * P, bits);
    }
}

__device__ __forceinline__ uint32_t op_kind(uint32_t o) { return o & 3u; }
__device__ __forceinline__ uint32_t op_len(uint32_t o) { return o >> 2; }
__device__ __forceinline__ uint32_t mk_op(uint32_t k, uint32_t l) { return k | l << 2; }

__device__ __forceinline__ uint32_t digits(uint32_t v) {
    uint32_t d = 1;
    while (v >= 10) { v /= 10; d++; }
    return d;
}

__global__ void __launch_bounds__(AT_THREADS) k_align_trace(AlnArgs a) {
    const uint32_t jid = blockIdx.x * AT_THREADS + threadIdx.x;
    if (jid >= a.n_jobs) return;
    const AlnJob J = a.jobs[jid];
    const int64_t w = a.w, W2 = 2 * w;
    const uint32_t n = J.tend - J.tstart, m = J.qend - J.qstart;
    const uint8_t* tb = a.tb + J.tb_off;
    uint32_t* ops = a.ops + J.op_off;
    const uint64_t* tw = a.rs.words + a.rs.word_off[J.tid];
    const QView qv = job_qview(a.rs, J);
    auto T = [&](uint64_t x) { return code_at(tw, J.tstart + (uint32_t)x); };
    auto Q = [&](uint64_t x) { return qv.code((uint32_t)x); };
    // ---- walk back from (n, m), run-length encoded (ops come out last to first)
    int64_t i = n, j = m;
    uint32_t st = 0, nops = 0, ck = 3, cn = 0;
    bool edge = false, bad = false;
    while (i > 0 || j > 0 || st != 0) {
        const int64_t k = j - ((int64_t)(((uint64_t)i * m) / n) - w);
        if (i < 0 || j < 0 || k < 0 || k >= W2) { bad = true; break; }  // cannot happen: every traced cell has a finite score
        if (k == 0 || k == W2 - 1) edge = true;
        const uint32_t b = tb[(uint64_t)i * W2 + k];
        uint32_t kind = 3;
        switch (st) {
            case 0: { const uint32_t s = b & 7u; if (s == 0) { kind = A_M; i--; j--; } else st = s; break; }
            case 1: kind = A_D; i--; st = (b >> 3 & 1u) ? 1u : 0u; break;
            case 2: kind = A_D; i--; st = (b >> 4 & 1u) ? 2u : 0u; break;
            case 3: kind = A_I; j--; st = (b >> 5 & 1u) ? 3u : 0u; break;
            default: kind = A_I; j--; st = (b >> 6 & 1u) ? 4u : 0u; break;
        }
        if (kind == 3) continue;
        if (kind == ck) { cn++; continue; }
        if (cn) ops[nops++] = mk_op(ck, cn);
        ck = kind;
        cn = 1;
    }
    if (cn) ops[nops++] = mk_op(ck, cn);
    for (uint32_t x = 0, y = nops - 1; x < y; x++, y--) { const uint32_t v = ops[x]; ops[x] = ops[y]; ops[y] = v; }
    // ---- fix_cigar: left-align every indel flanked by matches
    uint64_t tpos = 0, qpos = 0;
    for (uint32_t x = 0; x < nops; x++) {
        const uint32_t o = ops[x];
        if (op_kind(o) == A_M) { tpos += op_len(o); qpos += op_len(o); continue; }
        if (x > 0 && x + 1 < nops && op_kind(ops[x - 1]) == A_M && op_kind(ops[x + 1]) == A_M) {
            const uint32_t prev = op_len(ops[x - 1]), len = op_len(o);
            uint32_t l = 0;
            if (op_kind(o) == A_I) { while (l < prev && Q(qpos - 1 - l) == Q(qpos + len - 1 - l)) l++; }
            else { while (l < prev && T(tpos - 1 - l) == T(tpos + len - 1 - l)) l++; }
            if (l) { ops[x - 1] -= l << 2; ops[x + 1] += l << 2; tpos -= l; qpos -= l; }
        }
        if (op_kind(o) == A_I) qpos += op_len(o); else tpos += op_len(o);
    }
    // drop a leading gap op (and leading empty matches) into the shifts, then every empty op; merge equal neighbours
    uint32_t tsh = 0, qsh = 0, r = 0;
    bool start = true;
    for (uint32_t x = 0; x < nops; x++) {
        const uint32_t o = ops[x];
        if (start) {
            if (op_kind(o) == A_M) { if (!op_len(o)) continue; start = false; }
            else { start = false; if (op_kind(o) == A_I) qsh = op_len(o); else tsh = op_len(o); continue; }
        }
        if (!op_len(o)) continue;
        if (r && op_kind(ops[r - 1]) == op_kind(o)) ops[r - 1] += o & ~3u;
        else ops[r++] = o;
    }
    // ---- end gaps left over go into the shifts as well
    uint32_t f = 0, e = r, td = 0, ti = 0;
    while (f < e && op_kind(ops[f]) != A_M) { if (op_kind(ops[f]) == A_I) qsh += op_len(ops[f]); else tsh += op_len(ops[f]); f++; }
    while (e > f && op_kind(ops[e - 1]) != A_M) { if (op_kind(ops[e - 1]) == A_I) ti += op_len(ops[e - 1]); else td += op_len(ops[e - 1]); e--; }
    // ---- identical pairs inside M (32 bases at a time), text length
    uint32_t matches = 0, text = 0;
    uint64_t t = tsh, q = qsh;
    for (uint32_t x = f; x < e; x++) {
        const uint32_t o = ops[x], len = op_len(o);
        ops[x - f] = o;
        text += digits(len) + 1;
        if (op_kind(o) == A_I) { q += len; continue; }
        if (op_kind(o) == A_D) { t += len; continue; }
        for (uint32_t y = 0; y < len; y += 32) {
            const uint32_t c = min(32u, len - y);
            matches += c - __popcll(mismatch_groups(extract32(tw, J.tstart + (uint32_t)(t + y)), qv.chunk((uint32_t)(q + y)), c));
        }
        t += len;
        q += len;
    }
    AlnOut out;
    out.tstart = J.tstart + tsh;
    out.tend = J.tend - td;
    if (J.strand) { out.qstart = J.qstart + ti; out.qend = J.qend - qsh; }
    else { out.qstart = J.qstart + qsh; out.qend = J.qend - ti; }
    out.edge = bad ? 2u : edge ? 1u : 0u;
    out.matches = matches;
    out.n_ops = e - f;
    out.text_len = text;
    a.out[jid] = out;
}

// The CIGAR text of every job at a.text + a.text_off[job]
__global__ void __launch_bounds__(AT_THREADS) k_align_text(AlnArgs a) {
    const uint32_t jid = blockIdx.x * AT_THREADS + threadIdx.x;
    if (jid >= a.n_jobs) return;
    const uint32_t* ops = a.ops + a.jobs[jid].op_off;
    uint8_t* s = a.text + a.text_off[jid];
    const uint32_t no = a.out[jid].n_ops;
    for (uint32_t x = 0; x < no; x++) {
        uint32_t len = op_len(ops[x]);
        const uint32_t nd = digits(len);
        for (uint32_t k = nd; k-- > 0;) { s[k] = (uint8_t)('0' + len % 10); len /= 10; }
        s[nd] = "MID"[op_kind(ops[x])];
        s += nd + 1;
    }
}

}  // namespace

// Cells per lane for a band of 2w cells: 2w / 32 rounded up to a power of two (w a multiple of 16, at most ALN_MAX_W)
static uint32_t cells_per_lane(uint32_t w) {
    uint32_t p = 1;
    while (p * 32 < 2 * w) p <<= 1;
    return p;
}

void launch_align_fill(const AlnArgs& a, cudaStream_t st) {
    const uint32_t blocks = (a.n_jobs + AF_WARPS - 1) / AF_WARPS;
    switch (cells_per_lane(a.w)) {
        case 1: k_align_fill<1><<<blocks, AF_WARPS * 32, 0, st>>>(a); break;
        case 2: k_align_fill<2><<<blocks, AF_WARPS * 32, 0, st>>>(a); break;
        case 4: k_align_fill<4><<<blocks, AF_WARPS * 32, 0, st>>>(a); break;
        case 8: k_align_fill<8><<<blocks, AF_WARPS * 32, 0, st>>>(a); break;
        default: k_align_fill<16><<<blocks, AF_WARPS * 32, 0, st>>>(a); break;
    }
}

void launch_align_trace(const AlnArgs& a, cudaStream_t st) {
    k_align_trace<<<(a.n_jobs + AT_THREADS - 1) / AT_THREADS, AT_THREADS, 0, st>>>(a);
}

void launch_align_text(const AlnArgs& a, cudaStream_t st) {
    k_align_text<<<(a.n_jobs + AT_THREADS - 1) / AT_THREADS, AT_THREADS, 0, st>>>(a);
}

}  // namespace hb
