// reads_in.cu — k_reads_in: the reads of one launch, copied from the host read store (page-locked, device-mapped host memory,
// hb_attach_read_store) into the launch's batch region, so that the feature kernels find them through an ordinary ReadStoreView.
//
// A host-built list names every distinct read of the launch once, with its source offsets in the store and its destination
// offsets in the region; both sides keep every read's words and qualities 16-byte aligned and padded to a multiple of 16 bytes
// (zero words, quality 33), so a read is a run of whole 16-byte vectors.  One warp copies one read at a time: consecutive lanes
// load consecutive vectors (512 contiguous bytes per warp load), four loads in flight per lane before the first store, with a
// no-allocate / evict-first hint since the data is read once.  Lane 0 writes the read's entries of the region's word_off /
// qual_off tables, which stream order makes visible to the feature kernels.  Block 0 also writes the padding the uploaded store
// keeps around its reads (32 zero words and 256 bytes of 33 in front, 8 zero words and 16 bytes of 33 behind).
//
// The bound is PCIe: the grid is sized to keep about 256 KB of reads in flight, a few times the link's bandwidth-delay product,
// and no more, since the kernel shares the SMs with another lane's forward.
#include "common.cuh"
#include "forward.h"

namespace hb {

namespace {

constexpr int RI_THREADS = 256;
constexpr int RI_BLOCKS = 16;  // x 8 warps x 4 loads x 512 B = 256 KB in flight
constexpr int RI_UNROLL = 4;

__device__ __forceinline__ uint4 ld_stream(const uint4* p, uint64_t pol) {
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0, %1, %2, %3}, [%4], %5;"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(p), "l"(pol));
    return v;
}

// n 16-byte vectors from s to d by the 32 lanes of a warp
__device__ __forceinline__ void copy_vectors(const uint4* __restrict__ s, uint4* __restrict__ d, uint64_t n, uint32_t lane, uint64_t pol) {
    uint64_t k = lane;
    for (; k + 32 * (RI_UNROLL - 1) < n; k += 32 * RI_UNROLL) {
        uint4 v[RI_UNROLL];
#pragma unroll
        for (int u = 0; u < RI_UNROLL; u++) v[u] = ld_stream(s + k + 32 * u, pol);
#pragma unroll
        for (int u = 0; u < RI_UNROLL; u++) d[k + 32 * u] = v[u];
    }
    for (; k < n; k += 32) d[k] = ld_stream(s + k, pol);
}

__global__ void __launch_bounds__(RI_THREADS) k_reads_in(ReadsInArgs a) {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    const uint32_t lane = threadIdx.x & 31u;
    if (blockIdx.x == 0) {
        const uint32_t t = threadIdx.x;
        if (t < READS_FRONT_WORDS) a.words[t] = 0;
        if (t < READS_BACK_WORDS) a.words[READS_FRONT_WORDS + a.n_words + t] = 0;
        if (t < READS_FRONT_QUAL) a.qual[t] = QUAL_EMPTY;
        if (t < READS_BACK_QUAL) a.qual[READS_FRONT_QUAL + a.n_qual + t] = QUAL_EMPTY;
    }
    const uint32_t warps = gridDim.x * (RI_THREADS / 32);
    for (uint32_t i = blockIdx.x * (RI_THREADS / 32) + (threadIdx.x >> 5); i < a.n; i += warps) {
        const ReadCopy c = a.list[i];
        if (lane == 0) {
            a.word_off[c.rid] = c.dst_w;
            a.qual_off[c.rid] = c.dst_q;
        }
        copy_vectors((const uint4*)(a.src_words + c.src_w), (uint4*)(a.words + READS_FRONT_WORDS + c.dst_w), ((uint64_t)c.len + 63) / 64,
                     lane, pol);
        copy_vectors((const uint4*)(a.src_qual + c.src_q), (uint4*)(a.qual + READS_FRONT_QUAL + c.dst_q), ((uint64_t)c.len + 15) / 16,
                     lane, pol);
    }
}

}  // namespace

uint64_t launch_reads_in(const ReadsInArgs& a, cudaStream_t st, KTimer& kt) {
    kt.begin(K_LISTS);
    k_reads_in<<<RI_BLOCKS, RI_THREADS, 0, st>>>(a);
    kt.end();
    return 1;
}

}  // namespace hb
