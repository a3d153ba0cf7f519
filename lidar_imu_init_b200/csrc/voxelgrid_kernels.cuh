// voxelgrid_kernels.cuh -- scan voxel-grid downsample on the device (SURVEY.md section 8f row N2).
//
// Replaces `downSizeFilterSurf.filter(*feats_down_body)` (src/laserMapping.cpp:122,823,917-918), i.e. PCL's
// VoxelGrid<PointT>::applyFilter (PCL >= 1.8, pcl/filters/impl/voxel_grid.hpp -- third-party, not vendored in the
// reference): bounding box of the finite points, leaf index ijk = floor(p * inv_leaf) - min_b, linear index
// idx = i + j*dx + k*dx*dy, one output point per occupied leaf = float centroid (sum / count) of its points.
// PCL orders the output by idx and (std::sort, unstable) leaves the summation order inside a leaf unspecified; here
// the summation order is the input order (deterministic, bit-equal to the oracle's stable restatement, within one
// ulp per addend of any PCL build) and the output order is PCL's: ascending leaf index (radix sort of the unique leaf
// keys, sort_kernels.cuh) -- which is also the spatially coherent order the 5-NN kernel likes.
#pragma once
#include "common.cuh"
#include "map_kernels.cuh"
#include "sort_kernels.cuh"

struct VgParams {
    int min_b[3];
    int div_b[3];
    int mul1, mul2;   // divb_mul = (1, dx, dx*dy)
    int overflow;     // dx*dy*dz exceeds int32 (PCL: "Leaf size is too small"), or no finite point
    float inv_leaf;
};

__device__ __forceinline__ int li_f2ord(float f) {
    int i = __float_as_int(f);
    return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float li_ord2f(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }

// mm[0..2] = min (ordered ints), mm[3..5] = max; initialised to +inf / -inf by the host
__global__ void k_vg_minmax(const float4* __restrict__ pts, int n, int* __restrict__ mm) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    if (i < n) {
        float4 p = pts[i];
        if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
            lo[0] = hi[0] = p.x; lo[1] = hi[1] = p.y; lo[2] = hi[2] = p.z;
        }
    }
#pragma unroll
    for (int a = 0; a < 3; a++) {
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) {
            lo[a] = fminf(lo[a], __shfl_xor_sync(LI_FULL, lo[a], o));
            hi[a] = fmaxf(hi[a], __shfl_xor_sync(LI_FULL, hi[a], o));
        }
        if ((threadIdx.x & 31) == 0) {
            atomicMin(&mm[a], li_f2ord(lo[a]));
            atomicMax(&mm[3 + a], li_f2ord(hi[a]));
        }
    }
}

__global__ void k_vg_params(const int* __restrict__ mm, float leaf, VgParams* __restrict__ P) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    VgParams q;
    q.inv_leaf = 1.0f / leaf;   // Eigen::Array4f::Ones() / leaf_size (float)
    q.overflow = 0;
    long long d[3];
    double ext = 1.0;
    for (int a = 0; a < 3; a++) {
        float lo = li_ord2f(mm[a]), hi = li_ord2f(mm[3 + a]);
        if (!(lo <= hi)) {
            q.overflow = 1;
            lo = hi = 0.f;
        }
        ext *= floor((double)__fmul_rn(__fsub_rn(hi, lo), q.inv_leaf)) + 1.0;   // PCL's pre-check: dx*dy*dz must fit int32
        q.min_b[a] = (int)floorf(__fmul_rn(lo, q.inv_leaf));
        int mb = (int)floorf(__fmul_rn(hi, q.inv_leaf));
        d[a] = (long long)mb - (long long)q.min_b[a] + 1;
        q.div_b[a] = (int)d[a];
    }
    if (ext > 2147483647.0) q.overflow = 1;
    if (!q.overflow && d[0] * d[1] * d[2] > 2147483647ll) q.overflow = 1;
    q.mul1 = q.div_b[0];
    q.mul2 = q.div_b[0] * q.div_b[1];
    *P = q;
}

// link every finite point into the list of its leaf; imin = smallest point index of the leaf
__global__ void k_vg_link(const float4* __restrict__ pts, int n, const VgParams* __restrict__ Pp, VoxTmp V, int* __restrict__ imin,
                          int* __restrict__ next_of, int* __restrict__ slot_of, int* __restrict__ err) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    next_of[i] = -2;
    slot_of[i] = -1;
    const VgParams P = *Pp;
    if (P.overflow) return;
    float4 p = pts[i];
    if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z))) return;
    int i0 = (int)(floorf(__fmul_rn(p.x, P.inv_leaf)) - (float)P.min_b[0]);
    int i1 = (int)(floorf(__fmul_rn(p.y, P.inv_leaf)) - (float)P.min_b[1]);
    int i2 = (int)(floorf(__fmul_rn(p.z, P.inv_leaf)) - (float)P.min_b[2]);
    unsigned long long key = (unsigned long long)(unsigned)(i0 + i1 * P.mul1 + i2 * P.mul2);
    unsigned h = (unsigned)((key * 0x9E3779B97F4A7C15ull) >> 32) & V.mask;
    int slot = -1;
    for (unsigned t = 0; t <= V.mask; t++) {
        unsigned long long k = *reinterpret_cast<volatile unsigned long long*>(&V.keys[h]);
        if (k == key) { slot = (int)h; break; }
        if (k == LI_EMPTY_KEY) {
            unsigned long long old = atomicCAS(&V.keys[h], LI_EMPTY_KEY, key);
            if (old == LI_EMPTY_KEY || old == key) { slot = (int)h; break; }
        }
        h = (h + 1) & V.mask;
    }
    if (slot < 0) {
        atomicOr(err, 1);
        return;
    }
    slot_of[i] = slot;
    atomicMin(&imin[slot], i);
    next_of[i] = atomicExch(&V.head[slot], i);
}

__global__ void k_vg_clear(VoxTmp V, int* __restrict__ imin) {
    unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > V.mask) return;
    V.keys[i] = LI_EMPTY_KEY;
    V.head[i] = -1;
    imin[i] = 0x7fffffff;
}

// one (leaf index, first point index) pair per occupied leaf, in arbitrary order (sorted afterwards: keys are unique)
__global__ void k_vg_collect(VoxTmp V, const int* __restrict__ imin, unsigned* __restrict__ keys, unsigned* __restrict__ vals,
                             int* __restrict__ count) {
    unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > V.mask) return;
    if (V.head[i] < 0) return;
    int pos = atomicAdd(count, 1);
    keys[pos] = (unsigned)V.keys[i];
    vals[pos] = (unsigned)imin[i];
}

// one thread per leaf, leaves in ascending leaf index (PCL's output order): sum the leaf's points in input order. attr (optional):
// the attribute channel of the staged points {normal_x, normal_y, normal_z, intensity}, averaged the same way into out_attr
// (VoxelGrid with downsample_all_data_, the default: every field is a leaf mean; the curvature mean is never published)
__global__ void k_vg_centroid_sorted(const float4* __restrict__ pts, const unsigned* __restrict__ reps, const int* __restrict__ count,
                                     const int* __restrict__ slot_of, VoxTmp V, int* __restrict__ next_of, float4* __restrict__ out,
                                     int out_cap, int* __restrict__ err, const float4* __restrict__ attr, float4* __restrict__ out_attr) {
    int pos = blockIdx.x * blockDim.x + threadIdx.x;
    if (pos >= *count) return;
    if (pos >= out_cap) {
        atomicOr(err, 2);
        return;
    }
    // ascending input index. Short lists (the usual leaf): repeatedly take the smallest index greater than the last one -- k^2 loads but no
    // stores; long lists (near-sensor leaves of a dense raw scan): sort the links once (merge sort), then one walk
    int head = V.head[slot_of[reps[pos]]];
    float sx = 0.f, sy = 0.f, sz = 0.f;
    float ax = 0.f, ay = 0.f, az = 0.f, aw = 0.f;
    int cnt = 0;
    if (li_list_longer_than(head, next_of, LI_LIST_SELECT_MAX)) {
        head = li_list_sort_ascending(head, next_of);
        for (int cur = head; cur >= 0; cur = next_of[cur]) {
            float4 p = pts[cur];
            sx = __fadd_rn(sx, p.x);
            sy = __fadd_rn(sy, p.y);
            sz = __fadd_rn(sz, p.z);
            if (attr) {
                const float4 a = attr[cur];
                ax = __fadd_rn(ax, a.x); ay = __fadd_rn(ay, a.y); az = __fadd_rn(az, a.z); aw = __fadd_rn(aw, a.w);
            }
            cnt++;
        }
    } else {
        int last = -1;
        for (;;) {
            int cur = 0x7fffffff;
            for (int t = head; t >= 0; t = next_of[t])
                if (t > last && t < cur) cur = t;
            if (cur == 0x7fffffff) break;
            last = cur;
            float4 p = pts[cur];
            sx = __fadd_rn(sx, p.x);
            sy = __fadd_rn(sy, p.y);
            sz = __fadd_rn(sz, p.z);
            if (attr) {
                const float4 a = attr[cur];
                ax = __fadd_rn(ax, a.x); ay = __fadd_rn(ay, a.y); az = __fadd_rn(az, a.z); aw = __fadd_rn(aw, a.w);
            }
            cnt++;
        }
    }
    float c = (float)cnt;
    out[pos] = make_float4(__fdiv_rn(sx, c), __fdiv_rn(sy, c), __fdiv_rn(sz, c), 0.f);
    if (attr) out_attr[pos] = make_float4(__fdiv_rn(ax, c), __fdiv_rn(ay, c), __fdiv_rn(az, c), __fdiv_rn(aw, c));
}
