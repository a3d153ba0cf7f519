// sort_kernels.cuh -- small deterministic LSD radix sort of (key u32, value u32) pairs, 8 bits per pass.
//
// Used to emit the voxel-grid output in PCL's order (ascending leaf index, laserMapping.cpp:917-918 -> VoxelGrid),
// which is also a spatially coherent order for the 5-NN kernel (neighbouring scan points share bricks and walk the
// same shells). A few hundred thousand keys once per scan: simplicity and determinism matter more than peak speed.
// One warp owns a tile of RS_TILE consecutive keys and keeps their relative order (stable): match_any ranks the
// equal digits inside a 32-key row, a shared counter array carries the per-digit totals from row to row.
#pragma once
#include "common.cuh"

#define RS_TILE 1024

// The element count is n, or *n_dev when n_dev is given: the voxel grid and the frame cut learn their counts on the device and launch
// for the bound n (ntiles = ceil(n / RS_TILE)); the tiles past the real count then do no work.

// pass 1: per-tile digit histogram -> hist[digit * ntiles + tile]
__global__ void k_rs_hist(const unsigned* __restrict__ keys, int n, const int* __restrict__ n_dev, int shift, int ntiles, int* __restrict__ hist) {
    __shared__ int s_cnt[4][256];
    if (n_dev) n = *n_dev;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile = blockIdx.x * 4 + warp;
    for (int d = lane; d < 256; d += 32) s_cnt[warp][d] = 0;
    __syncwarp();
    if (tile < ntiles) {
        const int lo = tile * RS_TILE, hi = min(n, lo + RS_TILE);
        for (int i = lo + lane; i < hi; i += 32) atomicAdd(&s_cnt[warp][(keys[i] >> shift) & 255u], 1);
        __syncwarp();
        for (int d = lane; d < 256; d += 32) hist[d * ntiles + tile] = s_cnt[warp][d];
    }
}

// pass 2: exclusive scan of hist (256 * ntiles ints) by one block
__global__ void k_rs_scan(int m, int* __restrict__ a) {
    __shared__ int s_carry;
    __shared__ int s_w[32];
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (int base = 0; base < m; base += blockDim.x) {
        int i = base + threadIdx.x;
        int v = (i < m) ? a[i] : 0;
        int x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int y = __shfl_up_sync(LI_FULL, x, o);
            if ((threadIdx.x & 31) >= o) x += y;
        }
        if ((threadIdx.x & 31) == 31) s_w[threadIdx.x >> 5] = x;
        __syncthreads();
        if (threadIdx.x < 32) {
            int t = (threadIdx.x < (blockDim.x >> 5)) ? s_w[threadIdx.x] : 0;
            int z = t;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                int y = __shfl_up_sync(LI_FULL, z, o);
                if (threadIdx.x >= o) z += y;
            }
            s_w[threadIdx.x] = z - t;
        }
        __syncthreads();
        int excl = s_carry + s_w[threadIdx.x >> 5] + x - v;
        if (i < m) a[i] = excl;
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) s_carry = excl + v;
        __syncthreads();
    }
}

// pass 3: stable scatter
__global__ void k_rs_scatter(const unsigned* __restrict__ keys, const unsigned* __restrict__ vals, int n, const int* __restrict__ n_dev, int shift,
                             int ntiles, const int* __restrict__ hist, unsigned* __restrict__ keys_out, unsigned* __restrict__ vals_out) {
    __shared__ int s_off[4][256];
    if (n_dev) n = *n_dev;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile = blockIdx.x * 4 + warp;
    if (tile < ntiles)
        for (int d = lane; d < 256; d += 32) s_off[warp][d] = hist[d * ntiles + tile];
    __syncwarp();
    if (tile >= ntiles) return;
    const int lo = tile * RS_TILE, hi = min(n, lo + RS_TILE);
    for (int base = lo; base < hi; base += 32) {
        const int i = base + lane;
        const bool valid = i < hi;
        unsigned k = valid ? keys[i] : 0u, v = valid ? vals[i] : 0u;
        unsigned d = valid ? ((k >> shift) & 255u) : 256u + lane;   // invalid lanes get unique pseudo digits
        unsigned peers = __match_any_sync(LI_FULL, d);
        int rank = __popc(peers & ((1u << lane) - 1u));
        int off = 0;
        if (valid) off = s_off[warp][d] + rank;
        __syncwarp();
        if (valid && rank == 0) s_off[warp][d] += __popc(peers);   // one leader per digit updates the running offset
        __syncwarp();
        if (valid) {
            keys_out[off] = k;
            vals_out[off] = v;
        }
    }
}

// 64-bit keys (the cell keys of the map assessment, assess_kernels.cuh): the passes above run over the low words with the element
// index as the value, then this kernel fetches each element's high word by the carried index and the passes run again over the high
// words. Every pass is stable, so the result is ordered by (high word, low word, index).
__global__ void k_rs_gather_hi(const unsigned long long* __restrict__ keys64, const unsigned* __restrict__ vals, int n,
                               unsigned* __restrict__ keys_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) keys_out[i] = (unsigned)(keys64[vals[i]] >> 32);
}
