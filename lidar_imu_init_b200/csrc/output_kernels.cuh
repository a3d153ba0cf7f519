// output_kernels.cuh -- the node's published point clouds on the device (publish_frame_world, publish_frame_body,
// publish_effect_world and the pcd_save accumulation, src/laserMapping.cpp:561-636).
//
// Every cloud leaves as 48-byte pcl::PointXYZINormal records, 12 floats {x, y, z, 1, normal_x, normal_y, normal_z, 0, intensity,
// curvature, 0, 0}: the data of the PointCloud2 that pcl::toROSMsg makes of a PointCloudXYZI. pointBodyToWorld (:209-220) writes xyz
// and copies the normals and the intensity into a freshly constructed point, so the world-frame records carry curvature 0. The
// attribute channel of a cloud (float4 {normal_x, normal_y, normal_z, intensity} per point) may be absent: it then reads as zeros.
#pragma once
#include "common.cuh"
#include "preprocess_kernels.cuh"   // li_block_excl_scan, LI_FR_TILE

__device__ __forceinline__ void li_store_rec(float* __restrict__ out, int i, float x, float y, float z, float4 a, float curv) {
    float4* o = reinterpret_cast<float4*>(out) + 3 * (size_t)i;
    o[0] = make_float4(x, y, z, 1.f);
    o[1] = make_float4(a.x, a.y, a.z, 0.f);
    o[2] = make_float4(a.w, curv, 0.f, 0.f);
}

// publish_frame_world / pcd_save: pointBodyToWorld of every point (staged cloud or resident scan) into fresh records
__global__ void k_cloud_world(const float4* __restrict__ pts, const float4* __restrict__ attr, int n, PoseD P, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 p = pts[i];
    float wx, wy, wz;
    li_body_to_world(P, p.x, p.y, p.z, wx, wy, wz);
    li_store_rec(out, i, wx, wy, wz, attr ? attr[i] : make_float4(0.f, 0.f, 0.f, 0.f), 0.f);
}

// publish_frame_body: the staged (undistorted) point as it is, curvature = its time offset [ms]
__global__ void k_cloud_body(const float4* __restrict__ pts, const float4* __restrict__ attr, int n, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 p = pts[i];
    li_store_rec(out, i, p.x, p.y, p.z, attr ? attr[i] : make_float4(0.f, 0.f, 0.f, 0.f), p.w);
}

// frame_stage: the attribute channel of a sub-frame (intensity of the message, normals 0)
__global__ void k_attr_from_inten(const float* __restrict__ inten, int n, float4* __restrict__ attr) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    attr[i] = make_float4(0.f, 0.f, 0.f, inten[i]);
}

// publish_effect_world, step 1: selected points per block (blockDim.x == LI_FR_TILE); block 0 also zeroes tsum[gridDim.x], which the
// exclusive scan then turns into the total (effect_feat_num)
__global__ void k_eff_count(const unsigned char* __restrict__ sel, int n, int* __restrict__ tsum) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    int tot;
    li_block_excl_scan(i < n && sel[i] ? 1 : 0, &tot);
    if (threadIdx.x == 0) {
        tsum[blockIdx.x] = tot;
        if (blockIdx.x == 0) tsum[gridDim.x] = 0;
    }
}

// step 2 (tsum: exclusive per-block offsets): the order-preserving compaction of laserCloudOri (:1013-1020), the intensity the
// Jacobian loop leaves in it (sqrt(R_inv) with R_inv = 1000, :1050-1051), then pointBodyToWorld with the given pose
__global__ void k_eff_emit(const unsigned char* __restrict__ sel, int n, const int* __restrict__ tsum, const float4* __restrict__ body,
                           const float4* __restrict__ attr, PoseD P, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int f = i < n && sel[i] ? 1 : 0;
    int tot;
    const int pos = tsum[blockIdx.x] + li_block_excl_scan(f, &tot);
    if (!f) return;
    const float4 b = body[i];
    float wx, wy, wz;
    li_body_to_world(P, b.x, b.y, b.z, wx, wy, wz);
    float4 a = attr ? attr[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    a.w = (float)sqrt(1000.0);
    li_store_rec(out, pos, wx, wy, wz, a, 0.f);
}
