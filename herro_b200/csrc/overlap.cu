// overlap.cu — all-vs-all read overlaps (hb_find_overlaps, DESIGN.md §13): minimizer sketch, the index of the call's targets
// with its occurrence filter and hash table, the anchors of each query chunk, and their chains.
//
// k_ovl_sketch: one warp per read, 32 positions per step.  Each lane takes the k-mer ending at its position from two packed words
// with a funnel shift (extract32), hashes min(forward, reverse complement), and the non-skipped k-mers of the step are compacted by
// a ballot into a 64-slot ring in shared memory.  Each new k-mer that closes a window scans the window's w slots for its minimum
// (h, i); a selection is emitted when it differs from the previous window's, which the lanes read from their predecessor by a
// shuffle.  A count pass and, after a scan of the counts, a write pass.
// k_ovl_table: the open-addressing table from each unfiltered hash to its (offset, count) run in the sorted index entries.
// k_ovl_anchors: one thread per query minimizer: one probe run in the table, then the hash's entries, self hits skipped.  Count
// pass and write pass, like the sketch.
// k_ovl_chain: one warp per (query, target, strand) group; the lanes score 32 predecessors per step and a warp reduction on
// (score, b), larger b winning ties, gives the sequential dynamic programming's choice.  Then the end, the backtrack and the
// group's chain.
// The radix sorts, scans, run-length encodings and the selection of kept chains are CUB's.
#include <cub/cub.cuh>

#include "common.cuh"
#include "forward.h"

namespace hb {

namespace {

constexpr int SK_WARPS = 4;
constexpr int AN_THREADS = 256;
constexpr int CH_WARPS = 4;
constexpr int TB_THREADS = 256;

__device__ __forceinline__ uint64_t hash64(uint64_t key, uint64_t mask) {
    key = (~key + (key << 21)) & mask;
    key = key ^ key >> 24;
    key = ((key + (key << 3)) + (key << 8)) & mask;
    key = key ^ key >> 14;
    key = ((key + (key << 2)) + (key << 4)) & mask;
    key = key ^ key >> 28;
    key = (key + (key << 31)) & mask;
    return key;
}

__device__ __forceinline__ uint32_t lanemask_lt(int lane) { return (1u << lane) - 1u; }

// k_ovl_sketch: write == 0 counts each read's minimizers into count[r]; write == 1 writes them from offset[r]
__global__ void __launch_bounds__(SK_WARPS * 32) k_ovl_sketch(OvlSketchArgs a, int write) {
    __shared__ uint64_t sh_h[SK_WARPS][64];
    __shared__ uint32_t sh_p[SK_WARPS][64];  // i << 1 | z
    const int wp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t r = blockIdx.x * SK_WARPS + wp;
    if (r >= a.n) return;
    const uint32_t len = a.lens[r], k = a.k, w = a.w;
    const uint64_t* words = a.rs.words + a.rs.word_off[a.rids[r]];
    const uint64_t mask = (1ull << (2 * k)) - 1;
    const uint32_t shift = 64 - 2 * k;
    const uint64_t out0 = write ? a.offset[r] : 0;
    uint64_t* h_ = sh_h[wp];
    uint32_t* p_ = sh_p[wp];
    uint64_t cnt = 0, nout = 0;    // non-skipped k-mers so far; minimizers so far
    uint32_t carry = 0xffffffffu;  // the previous window's selection (none yet)
    for (uint32_t base = k - 1; base < len; base += 32) {
        const uint32_t i = base + lane;
        bool ok = false;
        uint64_t h = 0;
        uint32_t pz = 0;
        if (i < len) {
            const uint64_t e = extract32(words, i - k + 1) & mask;  // base u of the k-mer at bits 2u
            const uint64_t rc = e ^ mask;                          // its reverse complement, first base most significant
            uint64_t x = __brevll(e);
            x = ((x >> 1) & 0x5555555555555555ull) | ((x & 0x5555555555555555ull) << 1);
            const uint64_t f = x >> shift;                          // the k-mer, first base most significant
            if (f != rc) {
                ok = true;
                h = hash64(f < rc ? f : rc, mask);
                pz = i << 1 | (rc < f ? 1u : 0u);
            }
        }
        const uint32_t bal = __ballot_sync(HB_FULL, ok);
        const uint32_t rank = __popc(bal & lanemask_lt(lane));
        const uint64_t c = cnt + rank;
        if (ok) {
            h_[c & 63] = h;
            p_[c & 63] = pz;
        }
        __syncwarp();
        const bool has = ok && c + 1 >= w;
        uint64_t sh = 0;
        uint32_t sp = 0;
        if (has) {
            uint64_t b = c + 1 - w;
            sh = h_[b & 63];
            sp = p_[b & 63];
            for (b++; b <= c; b++) {
                const uint64_t hb = h_[b & 63];
                if (hb < sh) { sh = hb; sp = p_[b & 63]; }
            }
        }
        const uint32_t hbal = __ballot_sync(HB_FULL, has);
        const uint32_t before = hbal & lanemask_lt(lane);
        const uint32_t from = before ? 31 - __clz(before) : lane;
        const uint32_t prev_sel = __shfl_sync(HB_FULL, sp, from);
        const bool emit = has && sp != (before ? prev_sel : carry);
        const uint32_t ebal = __ballot_sync(HB_FULL, emit);
        if (write && emit) {
            const uint64_t o = out0 + nout + __popc(ebal & lanemask_lt(lane));
            a.key[o] = sh;
            a.val[o] = (uint64_t)r << 32 | sp;
        }
        nout += __popc(ebal);
        const uint32_t last_sel = __shfl_sync(HB_FULL, sp, hbal ? 31 - __clz(hbal) : 0);
        if (hbal) carry = last_sel;
        cnt += __popc(bal);
        __syncwarp();
    }
    if (!write && lane == 0) a.count[r] = nout;
}

__global__ void __launch_bounds__(TB_THREADS) k_ovl_table(OvlTableArgs a) {
    const uint32_t d = blockIdx.x * TB_THREADS + threadIdx.x;
    if (d >= a.n_d) return;
    const uint32_t occ = a.occ[d];
    if (occ > a.max_occ) {
        atomicAdd(a.n_filtered, 1u);
        return;
    }
    const uint64_t h = a.uniq[d];
    uint64_t s = h & a.mask;
    while (true) {
        const unsigned long long prev = atomicCAS((unsigned long long*)&a.keys[s], (unsigned long long)OVL_EMPTY, (unsigned long long)h);
        if (prev == OVL_EMPTY) break;
        s = (s + 1) & a.mask;
    }
    a.vals[s] = make_uint2(a.occ_off[d], occ);
}

// k_ovl_anchors: write == 0 counts each query minimizer's anchors into count[m]; write == 1 writes them from offset[m]
__global__ void __launch_bounds__(AN_THREADS) k_ovl_anchors(OvlAnchorArgs a, int write) {
    const uint64_t m = (uint64_t)blockIdx.x * AN_THREADS + threadIdx.x;
    if (m >= a.n_min) return;
    const uint64_t h = a.mkey[m];
    uint64_t s = h & a.mask;
    uint2 v = make_uint2(0, 0);
    while (true) {
        const uint64_t kk = __ldg(a.keys + s);
        if (kk == h) { v = __ldg(a.vals + s); break; }
        if (kk == OVL_EMPTY) break;
        s = (s + 1) & a.mask;
    }
    const uint64_t mv = a.mval[m];
    const uint32_t qc = (uint32_t)(mv >> 32), j = (uint32_t)mv >> 1, zq = (uint32_t)mv & 1;
    const uint32_t qrid = __ldg(a.q_rids + qc);
    uint64_t o = write ? a.offset[m] : 0, n = 0;
    for (uint32_t e = v.x; e < v.x + v.y; e++) {
        const uint64_t ev = __ldg(a.ent_val + e);
        const uint32_t t = (uint32_t)(ev >> 32);
        if (__ldg(a.target_rids + t) == qrid) continue;
        if (write) {
            const uint32_t i = (uint32_t)ev >> 1, st = ((uint32_t)ev & 1) ^ zq;
            const uint32_t y = st ? __ldg(a.q_lens + qc) + a.k - 2 - j : j;
            a.gkey[o] = (uint64_t)qc << 33 | (uint64_t)t << 1 | st;
            a.xy[o] = (uint64_t)i << 32 | y;
            o++;
        }
        n++;
    }
    if (!write) a.count[m] = n;
}

__device__ __forceinline__ int32_t gap_cost(uint32_t l, uint32_t k) {
    return l ? (int32_t)((uint64_t)k * l / 100) + (int32_t)((31 - __clz(l)) >> 1) : 0;
}

__global__ void __launch_bounds__(CH_WARPS * 32) k_ovl_chain(OvlChainArgs a) {
    const uint32_t g = blockIdx.x * CH_WARPS + (threadIdx.x >> 5);
    if (g >= a.n_groups) return;
    const int lane = threadIdx.x & 31;
    const uint32_t n = a.gcount[g];
    const uint32_t off = a.goff[g];
    OvlGroup out{};
    out.gkey = a.gkey[g];
    if (n < a.min_anchors) {
        if (lane == 0) a.out[g] = out;
        return;
    }
    if (lane == 0) atomicAdd(a.n_chained, 1u);
    const uint64_t* xy = a.xy + off;
    int32_t* f = a.f + off;
    int32_t* pred = a.pred + off;
    const int32_t k = (int32_t)a.k;
    for (uint32_t ai = 0; ai < n; ai++) {
        const uint64_t va = xy[ai];
        const uint32_t xa = (uint32_t)(va >> 32), ya = (uint32_t)va;
        const int64_t lo = ai > a.max_iter ? (int64_t)ai - a.max_iter : 0;
        int32_t bs = INT32_MIN;
        int32_t bb = -1;
        for (int64_t top = (int64_t)ai - 1; top >= lo; top -= 32) {
            const int64_t b = top - lane;
            bool stop = b < lo;
            if (!stop) {
                const uint64_t vb = xy[b];
                const uint32_t dx = xa - (uint32_t)(vb >> 32);
                const int64_t dy = (int64_t)ya - (uint32_t)vb;
                if (dx > a.max_gap) {
                    stop = true;
                } else if (dx > 0 && dy > 0 && dy <= a.max_gap) {
                    const int64_t l = (int64_t)dx > dy ? (int64_t)dx - dy : dy - (int64_t)dx;
                    if (l <= a.bandwidth) {
                        const int64_t dxy = (int64_t)dx < dy ? (int64_t)dx : dy;
                        const int32_t md = (int32_t)(dxy < k ? dxy : k);
                        const int32_t sc = f[b] + md - gap_cost((uint32_t)l, a.k);
                        if (sc > bs) { bs = sc; bb = (int32_t)b; }
                    }
                }
            }
            if (__any_sync(HB_FULL, stop)) break;
        }
#pragma unroll
        for (int d = 16; d; d >>= 1) {
            const int32_t os = __shfl_xor_sync(HB_FULL, bs, d), ob = __shfl_xor_sync(HB_FULL, bb, d);
            if (os > bs || (os == bs && ob > bb)) { bs = os; bb = ob; }
        }
        if (lane == 0) {
            f[ai] = bs > k ? bs : k;
            pred[ai] = bs > k ? bb : -1;
        }
        __syncwarp();
    }
    // the end: the largest f, the first on ties
    int32_t es = INT32_MIN;
    uint32_t ea = 0xffffffffu;
    for (uint32_t ai = lane; ai < n; ai += 32)
        if (f[ai] > es) { es = f[ai]; ea = ai; }
#pragma unroll
    for (int d = 16; d; d >>= 1) {
        const int32_t os = __shfl_xor_sync(HB_FULL, es, d);
        const uint32_t oa = __shfl_xor_sync(HB_FULL, ea, d);
        if (os > es || (os == es && oa < ea)) { es = os; ea = oa; }
    }
    if (lane) return;
    out.score = es;
    out.x_last = (uint32_t)(xy[ea] >> 32);
    out.y_last = (uint32_t)xy[ea];
    int64_t cov_lo = -1;
    uint32_t cov = 0, cnt = 0, first = ea;
    for (int32_t ai = (int32_t)ea; ai >= 0; ai = pred[ai]) {
        cnt++;
        first = (uint32_t)ai;
        const int64_t e = (int64_t)(xy[ai] >> 32) + 1, s = e - k;
        if (cov_lo < 0 || e <= cov_lo) cov += (uint32_t)(e - s);
        else if (s < cov_lo) cov += (uint32_t)(cov_lo - s);
        cov_lo = cov_lo < 0 ? s : min(cov_lo, s);
    }
    out.n_anchors = cnt;
    out.x_first = (uint32_t)(xy[first] >> 32);
    out.y_first = (uint32_t)xy[first];
    out.covered = cov;
    out.kept = es >= (int32_t)a.min_score && cnt >= a.min_anchors;
    a.out[g] = out;
}

struct IsKept {
    __host__ __device__ bool operator()(const OvlGroup& g) const { return g.kept != 0; }
};

}  // namespace

void launch_ovl_sketch(const OvlSketchArgs& a, bool write, cudaStream_t st) {
    if (a.n) k_ovl_sketch<<<(a.n + SK_WARPS - 1) / SK_WARPS, SK_WARPS * 32, 0, st>>>(a, write ? 1 : 0);
}

void launch_ovl_table(const OvlTableArgs& a, cudaStream_t st) {
    if (a.n_d) k_ovl_table<<<(a.n_d + TB_THREADS - 1) / TB_THREADS, TB_THREADS, 0, st>>>(a);
}

void launch_ovl_anchors(const OvlAnchorArgs& a, bool write, cudaStream_t st) {
    if (a.n_min) k_ovl_anchors<<<(unsigned)((a.n_min + AN_THREADS - 1) / AN_THREADS), AN_THREADS, 0, st>>>(a, write ? 1 : 0);
}

void launch_ovl_chain(const OvlChainArgs& a, cudaStream_t st) {
    if (a.n_groups) k_ovl_chain<<<(a.n_groups + CH_WARPS - 1) / CH_WARPS, CH_WARPS * 32, 0, st>>>(a);
}

// ---- CUB: with tmp == nullptr each call only sets `bytes`
cudaError_t ovl_exclusive_sum(void* tmp, size_t& bytes, uint64_t* d, uint64_t n, cudaStream_t st) {
    return cub::DeviceScan::ExclusiveSum(tmp, bytes, d, d, (int64_t)n, st);
}

cudaError_t ovl_exclusive_sum_u32(void* tmp, size_t& bytes, const uint32_t* in, uint32_t* out, uint32_t n, cudaStream_t st) {
    return cub::DeviceScan::ExclusiveSum(tmp, bytes, in, out, (int64_t)n, st);
}

cudaError_t ovl_sort_pairs(void* tmp, size_t& bytes, uint64_t* keys[2], uint64_t* vals[2], int& sel, uint64_t n, int end_bit,
                           cudaStream_t st) {
    cub::DoubleBuffer<uint64_t> dk(keys[sel], keys[sel ^ 1]), dv(vals[sel], vals[sel ^ 1]);
    const cudaError_t e = cub::DeviceRadixSort::SortPairs(tmp, bytes, dk, dv, (int64_t)n, 0, end_bit, st);
    if (tmp && e == cudaSuccess && dk.Current() != keys[sel]) sel ^= 1;
    return e;
}

cudaError_t ovl_sort_u32(void* tmp, size_t& bytes, const uint32_t* in, uint32_t* out, uint32_t n, cudaStream_t st) {
    return cub::DeviceRadixSort::SortKeys(tmp, bytes, in, out, (int64_t)n, 0, 32, st);
}

cudaError_t ovl_runs(void* tmp, size_t& bytes, const uint64_t* in, uint64_t* uniq, uint32_t* counts, uint32_t* n_runs, uint64_t n,
                     cudaStream_t st) {
    return cub::DeviceRunLengthEncode::Encode(tmp, bytes, in, uniq, counts, n_runs, (int64_t)n, st);
}

cudaError_t ovl_select_kept(void* tmp, size_t& bytes, const OvlGroup* in, OvlGroup* out, uint32_t* n_sel, uint32_t n, cudaStream_t st) {
    return cub::DeviceSelect::If(tmp, bytes, in, out, n_sel, (int64_t)n, IsKept(), st);
}

}  // namespace hb
