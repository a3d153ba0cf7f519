// preprocess_kernels.cuh -- the cut-frame preprocess on the device (Preprocess::process_cut_frame_livox / _pcl2,
// src/preprocess.cpp:50-335): driver message -> decoded, filtered, time-sorted sub-frames, re-timed to their own start.
//
// The reference walks the message sequentially; every sequential dependency has a parallel form here:
//   * the Livox point-filter counter (valid_point_num) is an inclusive scan of the validity flags;
//   * the duplicate test against pl_full[i-1] needs only whether point i-1 was taken, which follows from the same count;
//   * the constant-rotation model of spinning sensors without a time field is per ring: after a stable sort of the survivors by
//     ring, a point is wrapped (+360/omega) iff it lies at or after the first descent of the ring's base times (once wrapped, a
//     time is >= float(360/omega) >= every later base; the one exception, a later base equal to float(360/omega), is detected and
//     the ring's loop is then run as the reference writes it);
//   * std::sort by curvature is the stable radix sort of sort_kernels.cuh on the float time flipped to an ordered u32 (a valid
//     outcome of std::sort; -0 and +0 compare equal);
//   * the cut itself is a chain over at most required_cut_num boundaries: one thread.
// All arithmetic keeps the reference's float / double mix (the library builds with --fmad=false).
#pragma once
#include "common.cuh"
#include "sort_kernels.cuh"

#define LI_FR_TILE 1024   // elements per block of the scan / compaction kernels (blockDim.x)

struct FrameSub {
    double lfet;   // last_frame_end_time at the start of the sub-frame [ms]
    float end_ms;  // re-timed curvature of its last point
    int lo;        // first sorted index
    int n;         // points
    int pad;
};
struct FrameTable {
    int V;      // valid_pcl_size (points after the filters)
    int nsub;   // sub-frames produced
    int err;    // bit 0: ring >= 128 in the rotation model; bit 1: the rotation model needs its sequential loop (k_fr_yaw_chain)
    int pad;
    FrameSub sub[LIINIT_FRAME_MAX_CUT];
};

struct Pcl2Dev {
    int step, ox, oy, oz, oi, ot, orr;
    int type;
    int yaw;      // offset times from the constant-rotation model
    double ts0;   // Pandar: timestamp of point 0
};

__device__ __forceinline__ unsigned li_ld_u32(const unsigned char* p) {
    return (unsigned)p[0] | ((unsigned)p[1] << 8) | ((unsigned)p[2] << 16) | ((unsigned)p[3] << 24);
}
__device__ __forceinline__ float li_ld_f32(const unsigned char* p) { return __uint_as_float(li_ld_u32(p)); }
__device__ __forceinline__ double li_ld_f64(const unsigned char* p) {
    const unsigned long long v = (unsigned long long)li_ld_u32(p) | ((unsigned long long)li_ld_u32(p + 4) << 32);
    return __longlong_as_double((long long)v);
}

// sort key of a float time: ascending float order as unsigned order, -0 == +0
__device__ __forceinline__ unsigned li_time_key(float t) {
    unsigned u = __float_as_uint(t);
    if (u == 0x80000000u) u = 0u;
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// exclusive scan of one int per thread over the block (blockDim.x == LI_FR_TILE); *total = the block's sum
__device__ int li_block_excl_scan(int v, int* total) {
    __shared__ int s_w[32];
    __shared__ int s_tot;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int y = __shfl_up_sync(LI_FULL, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) s_w[warp] = x;
    __syncthreads();
    if (warp == 0) {
        int t = (lane < (int)(blockDim.x >> 5)) ? s_w[lane] : 0;
        int z = t;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int y = __shfl_up_sync(LI_FULL, z, o);
            if (lane >= o) z += y;
        }
        s_w[lane] = z - t;
        if (lane == 31) s_tot = z;
    }
    __syncthreads();
    const int r = s_w[warp] + x - v;
    *total = s_tot;
    __syncthreads();
    return r;
}

// ---- Livox CustomMsg ----------------------------------------------------------------------------------------------------
// record: u32 offset_time @0, f32 x y z @4 8 12, u8 reflectivity @16, tag @17, line @18
__device__ __forceinline__ bool li_lvx_valid(const unsigned char* in, int stride, int i, int nscans) {
    if (i < 1) return false;   // the loop starts at 1
    const unsigned char* r = in + (size_t)i * stride;
    const unsigned tag = r[17] & 0x30u;
    return (int)r[18] < nscans && (tag == 0x10u || tag == 0x00u);
}

// flag[i] = valid; tsum[block] = number of valid points of the block
__global__ void k_fr_lvx_valid(const unsigned char* __restrict__ in, int stride, int n, int nscans, int* __restrict__ flag,
                               int* __restrict__ tsum) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int v = (i < n && li_lvx_valid(in, stride, i, nscans)) ? 1 : 0;
    if (i < n) flag[i] = v;
    int tot;
    li_block_excl_scan(v, &tot);
    if (threadIdx.x == 0) tsum[blockIdx.x] = tot;
}

// tsum: exclusive per-block offsets of the valid count. Decodes the taken points, applies the blind and duplicate tests;
// flag[i] = kept, tsum2[block] = kept points of the block.
__global__ void k_fr_lvx_keep(const unsigned char* __restrict__ in, int stride, int n, int nscans, int pfn, double blind2,
                              const int* __restrict__ tsum, int* __restrict__ flag, float4* __restrict__ dec, float* __restrict__ inten,
                              int* __restrict__ tsum2) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int v = i < n ? flag[i] : 0;
    int tot;
    const int cnt = tsum[blockIdx.x] + li_block_excl_scan(v, &tot) + v;   // valid_point_num after point i
    int keep = 0;
    if (v && cnt % pfn == 0) {
        const unsigned char* r = in + (size_t)i * stride;
        const float x = li_ld_f32(r + 4), y = li_ld_f32(r + 8), z = li_ld_f32(r + 12);
        const float curv = (float)li_ld_u32(r) / float(1000000);
        dec[i] = make_float4(x, y, z, curv);
        inten[i] = (float)r[16];
        const double dist = x * x + y * y + z * z;   // float arithmetic, widened
        if (!(dist < blind2)) {
            // pl_full[i-1]: the previous raw point if it was taken (blind or not), else the zero point of pl_full.resize
            float px = 0.f, py = 0.f, pz = 0.f;
            if (li_lvx_valid(in, stride, i - 1, nscans) && (cnt - 1) % pfn == 0) {
                const unsigned char* q = r - stride;
                px = li_ld_f32(q + 4); py = li_ld_f32(q + 8); pz = li_ld_f32(q + 12);
            }
            // abs() of a float is the float overload (using namespace std), compared in double
            keep = ((double)fabsf(x - px) > 1e-7) || ((double)fabsf(y - py) > 1e-7) || ((double)fabsf(z - pz) > 1e-7);
        }
    }
    if (i < n) flag[i] = keep;
    int kt;
    li_block_excl_scan(keep, &kt);
    if (threadIdx.x == 0) tsum2[blockIdx.x] = kt;
}

// ---- PointCloud2 --------------------------------------------------------------------------------------------------------
// Decodes point i (absent fields read 0, as fromROSMsg leaves them), applies the time rule, the blind / NaN test and -- with
// given times -- the point filter and the ring limit: flag[i] = kept. In the rotation model flag[i] = survived the blind / NaN
// test, key[i] = its ring (the rotation kernels decide the rest). tsum[block] = flags of the block.
__global__ void k_fr_pcl2_decode(const unsigned char* __restrict__ in, int n, Pcl2Dev L, int nscans, int pfn, double blind2, double stamp,
                                 int* __restrict__ flag, float4* __restrict__ dec, float* __restrict__ inten, unsigned* __restrict__ key,
                                 int* __restrict__ tsum, int* __restrict__ err) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    int f = 0;
    if (i < n) {
        const unsigned char* r = in + (size_t)i * L.step;
        const float x = L.ox >= 0 ? li_ld_f32(r + L.ox) : 0.f;
        const float y = L.oy >= 0 ? li_ld_f32(r + L.oy) : 0.f;
        const float z = L.oz >= 0 ? li_ld_f32(r + L.oz) : 0.f;
        float in_v = 0.f, curv = 0.f;
        unsigned ring = 0;
        if (L.type == 6) in_v = L.oi >= 0 ? (float)r[L.oi] : 0.f;
        else in_v = L.oi >= 0 ? li_ld_f32(r + L.oi) : 0.f;
        if (L.orr >= 0) ring = L.type == 3 ? (unsigned)r[L.orr] : ((unsigned)r[L.orr] | ((unsigned)r[L.orr + 1] << 8));
        if (L.type == 2) {
            const float t = L.ot >= 0 ? li_ld_f32(r + L.ot) : 0.f;
            curv = (float)(t * 1000.0);
        } else if (L.type == 3) {
            const unsigned t = L.ot >= 0 ? li_ld_u32(r + L.ot) : 0u;
            curv = (float)(t / 1e6);
        } else if (L.type == 5) {
            const double t = L.ot >= 0 ? li_ld_f64(r + L.ot) : 0.0;
            curv = (float)((t - L.ts0) * 1000);
        } else {
            const double t = L.ot >= 0 ? li_ld_f64(r + L.ot) : 0.0;
            curv = (float)((t - stamp + 0.1) * 1000.0);
        }
        dec[i] = make_float4(x, y, z, curv);
        inten[i] = in_v;
        const double dist = x * x + y * y + z * z;
        const bool survive = !(dist < blind2 || x != x || y != y || z != z);
        if (L.yaw) {
            f = survive;
            key[i] = ring < 255u ? ring : 255u;
            if (survive && ring >= 128u) atomicOr(err, 1);
        } else {
            f = survive && i % pfn == 0 && (int)ring < nscans;
        }
        flag[i] = f;
    }
    int tot;
    li_block_excl_scan(f, &tot);
    if (threadIdx.x == 0) tsum[blockIdx.x] = tot;
}

__device__ __forceinline__ double li_yaw_deg(float x, float y) {
    // atan2 of two floats is std::atan2(float, float); the device evaluates it in double and rounds once
    const float a = (float)atan2((double)y, (double)x);
    return (double)a * 57.2957;
}

__device__ __forceinline__ float li_yaw_base(double yaw, double yaw_fp) {
    const double omega_l = 3.61;
    return yaw <= yaw_fp ? (float)((yaw_fp - yaw) / omega_l) : (float)((yaw_fp - yaw + 360.0) / omega_l);
}

// rotation model, step 1: the yaw of every survivor (ring-sorted: key = ring, val = raw index) and the first position of each ring
__global__ void k_fr_yaw_first(const unsigned* __restrict__ key, const unsigned* __restrict__ val, const int* __restrict__ n_dev,
                               const float4* __restrict__ dec, double* __restrict__ yaw, int* __restrict__ ring_first,
                               int* __restrict__ ring_desc) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= *n_dev) return;
    const float4 q = dec[val[p]];
    yaw[p] = li_yaw_deg(q.x, q.y);
    const unsigned r = key[p];
    if (p == 0 || key[p - 1] != r) {
        ring_first[r] = p;
        ring_desc[r] = 0x7fffffff;
    }
}

// step 2: base time of every survivor (0 for the first point of a ring), and the first descent of each ring
__global__ void k_fr_yaw_base(const unsigned* __restrict__ key, const int* __restrict__ n_dev, const double* __restrict__ yaw,
                              const int* __restrict__ ring_first, float* __restrict__ base, int* __restrict__ ring_desc) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= *n_dev) return;
    const unsigned r = key[p];
    const int pf = ring_first[r];
    float b = 0.f;
    if (p != pf) {
        const double yaw_fp = yaw[pf];
        b = li_yaw_base(yaw[p], yaw_fp);
        const float bprev = p - 1 != pf ? li_yaw_base(yaw[p - 1], yaw_fp) : 0.f;   // time_last before any wrap
        if (b < bprev) atomicMin(&ring_desc[r], p);
    }
    base[p] = b;
}

// step 3: final times, the point filter and the ring limit; the first point of a ring is dropped. flag / dec by raw index.
// After the first descent the reference wraps a point iff base < time_last, and time_last >= float(360/omega) >= base there: the
// closed form "wrapped" fails only for a base equal to float(360/omega). Such a point sets err bit 1; k_fr_yaw_chain then redoes
// the times of every ring sequentially.
__global__ void k_fr_yaw_final(const unsigned* __restrict__ key, const unsigned* __restrict__ val, const int* __restrict__ n_dev,
                               const float* __restrict__ base, const int* __restrict__ ring_first, const int* __restrict__ ring_desc,
                               int nscans, int pfn, float4* __restrict__ dec, int* __restrict__ flag, int* __restrict__ err) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= *n_dev) return;
    const unsigned r = key[p];
    const int i = (int)val[p];
    if (p == ring_first[r]) {
        flag[i] = 0;
        return;
    }
    float t = base[p];
    if (p >= ring_desc[r]) {
        if (p > ring_desc[r] && t == (float)(360.0 / 3.61)) atomicOr(err, 2);
        t = (float)((double)t + 360.0 / 3.61);
    }
    dec[i].w = t;
    flag[i] = i % pfn == 0 && (int)r < nscans;
}

// the reference's per-ring loop over the stored bases, one thread per ring; runs only when k_fr_yaw_final set err bit 1
__global__ void k_fr_yaw_chain(const unsigned* __restrict__ key, const unsigned* __restrict__ val, const int* __restrict__ n_dev,
                               const float* __restrict__ base, const int* __restrict__ ring_first, const int* __restrict__ err,
                               float4* __restrict__ dec) {
    const unsigned r = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = *n_dev;
    if (!(*err & 2) || r >= 256u) return;
    const int pf = ring_first[r];
    if (pf < 0 || pf >= n || key[pf] != r || (pf > 0 && key[pf - 1] == r)) return;   // ring absent (stale entry)
    float time_last = 0.f;
    for (int p = pf + 1; p < n && key[p] == r; p++) {
        float t = base[p];
        if (t < time_last) t = (float)((double)t + 360.0 / 3.61);
        dec[val[p]].w = t;
        time_last = t;
    }
}

// tsum[block] = flags of the block
__global__ void k_fr_tile_count(const int* __restrict__ flag, int n, int* __restrict__ tsum) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    int tot;
    li_block_excl_scan(i < n ? flag[i] : 0, &tot);
    if (threadIdx.x == 0) tsum[blockIdx.x] = tot;
}

// order-preserving compaction of the flagged points into (key, raw index) pairs; key = key_src[i], or the time key of dec[i].w
// when key_src is NULL. tsum: exclusive per-block offsets. *n_out = number of flagged points.
__global__ void k_fr_compact(const int* __restrict__ flag, int n, const int* __restrict__ tsum, const float4* __restrict__ dec,
                             const unsigned* __restrict__ key_src, unsigned* __restrict__ keys, unsigned* __restrict__ vals, int* __restrict__ n_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int f = i < n ? flag[i] : 0;
    int tot;
    const int pos = tsum[blockIdx.x] + li_block_excl_scan(f, &tot);
    if (f) {
        keys[pos] = key_src ? key_src[i] : li_time_key(dec[i].w);
        vals[pos] = (unsigned)i;
    }
    if (i == n - 1) *n_out = pos + f;
}

// the cut (preprocess.cpp:86-112, 307-334): one thread walks the required_cut_num boundaries. Sub-frame k holds the sorted indices
// (t_{k-1}, t_k], t_k = int((k+1) V / R) - 1 (unsigned arithmetic, as the reference), t_{-1} = 0: sorted index 0 is dropped. A
// target <= 0 never matches the running count, so V < 2R gives no sub-frame at all; otherwise the R targets increase by >= 2.
__global__ void k_fr_bounds(const unsigned* __restrict__ vals, const float4* __restrict__ dec, int R, double S, FrameTable* __restrict__ T) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    const unsigned V = (unsigned)T->V;
    if ((T->err & 1) || (int)(V / (unsigned)R) - 1 <= 0) {
        T->nsub = 0;
        return;
    }
    double lfet = S;
    int prev = 0;
    for (int k = 0; k < R; k++) {
        const int t = (int)((unsigned)(k + 1) * V / (unsigned)R) - 1;
        const float end = (float)((double)dec[vals[t]].w + (S - lfet));
        T->sub[k].lfet = lfet;
        T->sub[k].end_ms = end;
        T->sub[k].lo = prev + 1;
        T->sub[k].n = t - prev;
        lfet += (double)end;
        prev = t;
    }
    T->nsub = R;
}

// re-time and gather sorted index j into the message slot at j - 1: {x, y, z, curvature} + intensity
__global__ void k_fr_gather(const unsigned* __restrict__ vals, const float4* __restrict__ dec, const float* __restrict__ inten, double S,
                            const FrameTable* __restrict__ T, float4* __restrict__ out, float* __restrict__ out_i) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x + 1;
    const int ns = T->nsub;
    if (ns == 0) return;
    if (j >= T->sub[ns - 1].lo + T->sub[ns - 1].n) return;
    int a = 0, b = ns - 1;   // last sub-frame with lo <= j
    while (a < b) {
        const int m = (a + b + 1) >> 1;
        if (T->sub[m].lo <= j) a = m;
        else b = m - 1;
    }
    const int i = (int)vals[j];
    const float4 p = dec[i];
    out[j - 1] = make_float4(p.x, p.y, p.z, (float)((double)p.w + (S - T->sub[a].lfet)));
    out_i[j - 1] = inten[i];
}
