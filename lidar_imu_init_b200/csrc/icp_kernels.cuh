// icp_kernels.cuh -- plane fit + residual + Jacobian row + HtH/Htr reduction (one scan point per lane).
//
// Replaces laserMapping.cpp:989-1071 (+ the dense reduction of :1080) and esti_plane (common_lib.h:236-269).
// The 5-NN that feeds it lives in knn_kernels.cuh. DESIGN.md section 5 has the derivations.
//
//   fp64 column-pivoted Householder LSQ of the 5x3 system, residual, gating, Jacobian row;
//   warp reduce-scatter of the 92 (imu) / 29 (lidar-only) accumulators; per-block partials and a
//   fixed-order final reduction by the last block (bit-reproducible).
#pragma once
#include "common.cuh"

#ifndef LI_PLANE_MIN_BLOCKS
#define LI_PLANE_MIN_BLOCKS 2
#endif

// ----------------------------------------------------------------------------------------------
// Phase 2 math (per scan point, fp64)

// min ||A x - b||, A 5x3 (rows = neighbours), b = -1: column-pivoted Householder QR (the method behind
// Eigen's colPivHouseholderQr().solve, common_lib.h:252).
__device__ __forceinline__ void lsq5x3(double (&A)[5][3], double (&x)[3]) {
    double b[5] = {-1.0, -1.0, -1.0, -1.0, -1.0};
    int p0 = 0, p1 = 1, p2 = 2;
    double maxn = 0.0;
    {
        double c0 = 0, c1 = 0, c2 = 0;
#pragma unroll
        for (int i = 0; i < 5; i++) {
            c0 += A[i][0] * A[i][0];
            c1 += A[i][1] * A[i][1];
            c2 += A[i][2] * A[i][2];
        }
        maxn = fmax(c0, fmax(c1, c2));
    }
    const double eps = 2.220446049250313e-16;
    const double sq = sqrt(maxn) * eps;
    const double thresh = sq * sq / 5.0;
    int rank = 3;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        if (rank < 3) continue;   // uniform per lane; remaining steps skipped once rank-deficient
        // column norms of the trailing block, pick the first maximum
        double cn[3] = {-1.0, -1.0, -1.0};
#pragma unroll
        for (int j = 0; j < 3; j++) {
            if (j >= k) {
                double s = 0;
#pragma unroll
                for (int i = 0; i < 5; i++)
                    if (i >= k) s += A[i][j] * A[i][j];
                cn[j] = s;
            }
        }
        int p = k;
        double best = cn[k];
#pragma unroll
        for (int j = 0; j < 3; j++) {
            if (j > k && cn[j] > best) {
                best = cn[j];
                p = j;
            }
        }
        if (best < thresh * (double)(5 - k)) {   // Eigen: biggest_col_sq_norm < threshold_helper * (rows - k)
            rank = k;
            continue;
        }
        if (p != k) {
            // swap columns k and p (static indices via unrolled selects)
#pragma unroll
            for (int j = 0; j < 3; j++) {
                if (j > k && j == p) {
#pragma unroll
                    for (int i = 0; i < 5; i++) {
                        double tmp = A[i][k];
                        A[i][k] = A[i][j];
                        A[i][j] = tmp;
                    }
                }
            }
            // permutation bookkeeping
            int pk = (k == 0) ? p0 : ((k == 1) ? p1 : p2);
            int pp = (p == 0) ? p0 : ((p == 1) ? p1 : p2);
            if (k == 0) p0 = pp; else if (k == 1) p1 = pp; else p2 = pp;
            if (p == 0) p0 = pk; else if (p == 1) p1 = pk; else p2 = pk;
        }
        double alpha = A[k][k];
        double tail = 0;
#pragma unroll
        for (int i = 0; i < 5; i++)
            if (i > k) tail += A[i][k] * A[i][k];
        if (tail != 0.0) {
            double nrm = sqrt(alpha * alpha + tail);
            double beta = (alpha >= 0) ? -nrm : nrm;
            double tau = (beta - alpha) / beta;
            double scale = 1.0 / (alpha - beta);
            double v[5];
#pragma unroll
            for (int i = 0; i < 5; i++) v[i] = (i == k) ? 1.0 : ((i > k) ? A[i][k] * scale : 0.0);
            A[k][k] = beta;
#pragma unroll
            for (int i = 0; i < 5; i++)
                if (i > k) A[i][k] = 0.0;
#pragma unroll
            for (int j = 0; j < 3; j++) {
                if (j > k) {
                    double s = 0;
#pragma unroll
                    for (int i = 0; i < 5; i++)
                        if (i >= k) s += v[i] * A[i][j];
                    s *= tau;
#pragma unroll
                    for (int i = 0; i < 5; i++)
                        if (i >= k) A[i][j] -= s * v[i];
                }
            }
            double s = 0;
#pragma unroll
            for (int i = 0; i < 5; i++)
                if (i >= k) s += v[i] * b[i];
            s *= tau;
#pragma unroll
            for (int i = 0; i < 5; i++)
                if (i >= k) b[i] -= s * v[i];
        }
    }
    double y0 = 0, y1 = 0, y2 = 0;
    if (rank >= 3) y2 = b[2] / A[2][2];
    if (rank >= 2) y1 = (b[1] - A[1][2] * y2) / A[1][1];
    if (rank >= 1) y0 = (b[0] - A[0][1] * y1 - A[0][2] * y2) / A[0][0];
    // x[perm[j]] = y[j]
    x[0] = (p0 == 0) ? y0 : ((p1 == 0) ? y1 : y2);
    x[1] = (p0 == 1) ? y0 : ((p1 == 1) ? y1 : y2);
    x[2] = (p0 == 2) ? y0 : ((p1 == 2) ? y1 : y2);
}

// esti_plane<double>(pca_result, point, 0.1f) (common_lib.h:236-269): plane (pa, pb, pc, pd) through the five neighbours
// (uncentred f32 -> f64 rows, A x = -1), unit normal; valid iff every neighbour lies within 0.1 of it.
__device__ __forceinline__ bool esti_plane_d(const float4 (&nb)[5], double& pa, double& pb, double& pc, double& pd) {
    double A[5][3];
#pragma unroll
    for (int j = 0; j < 5; j++) {
        A[j][0] = (double)nb[j].x;
        A[j][1] = (double)nb[j].y;
        A[j][2] = (double)nb[j].z;
    }
    double nv[3];
    lsq5x3(A, nv);
    double nn = sqrt(nv[0] * nv[0] + nv[1] * nv[1] + nv[2] * nv[2]);
    pa = nv[0] / nn; pb = nv[1] / nn; pc = nv[2] / nn; pd = 1.0 / nn;
    bool ok = true;
#pragma unroll
    for (int j = 0; j < 5; j++) {
        double e = fabs(pa * (double)nb[j].x + pb * (double)nb[j].y + pc * (double)nb[j].z + pd);
        if (!(e <= 0.1)) ok = false;    // reference: reject if > threshold (NaN also rejects via !(<=)... see note)
    }
    // note: the reference tests `fabs(..) > threshold -> return false`; a NaN plane passes that test there and is
    // rejected later by `s > 0.9` being false. Both forms reject NaN; finite cases are identical.
    return ok;
}

// test hook (liinit_debug_esti_plane): esti_plane for n independent neighbour sets
__global__ void k_debug_esti_plane(const float* __restrict__ nb_xyz, int n, double* __restrict__ pabcd, unsigned char* __restrict__ valid) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float4 nb[5];
#pragma unroll
    for (int j = 0; j < 5; j++) nb[j] = make_float4(nb_xyz[(size_t)i * 15 + 3 * j], nb_xyz[(size_t)i * 15 + 3 * j + 1], nb_xyz[(size_t)i * 15 + 3 * j + 2], 1.f);
    double pa, pb, pc, pd;
    const bool ok = esti_plane_d(nb, pa, pb, pc, pd);
    pabcd[(size_t)i * 4] = pa; pabcd[(size_t)i * 4 + 1] = pb; pabcd[(size_t)i * 4 + 2] = pc; pabcd[(size_t)i * 4 + 3] = pd;
    valid[i] = ok ? 1 : 0;
}

// Number of accumulators: upper triangle of HtH + Htr + sum r^2 + count, padded to a multiple of 32.
template <bool IMU>
struct AccLayout {
    static constexpr int NC = IMU ? 12 : 6;
    static constexpr int NT = NC * (NC + 1) / 2;        // 78 / 21
    static constexpr int NV = NT + NC + 2;              // 92 / 29
    static constexpr int V = ((NV + 31) / 32) * 32;     // 96 / 32
    static constexpr int K = V / 32;                    // 3 / 1
};

// esti_plane + residual + gate + Jacobian row for one scan point (laserMapping.cpp:995-1010,1035-1071).
// Returns selected; fills row[NC] and r = meas = -pd2 (zeros when not selected).
template <bool IMU>
__device__ __forceinline__ bool plane_and_row(const PoseD& P, float bxf, float byf, float bzf, float wx, float wy, float wz,
                                              const float4 (&nb)[5], float4& normvec_out,
                                              double (&row)[AccLayout<IMU>::NC], double& r) {
    typedef AccLayout<IMU> L;
#pragma unroll
    for (int i = 0; i < L::NC; i++) row[i] = 0.0;
    r = 0.0;
    double pa, pb, pc, pd;
    if (!esti_plane_d(nb, pa, pb, pc, pd)) return false;
    float pd2 = (float)(pa * (double)wx + pb * (double)wy + pc * (double)wz + pd);
    double bx = (double)bxf, by = (double)byf, bz = (double)bzf;
    double pn = sqrt(bx * bx + by * by + bz * bz);
    float s = (float)(1.0 - 0.9 * (double)fabsf(pd2) / sqrt(pn));
    if (!((double)s > 0.9)) return false;
    float nxf = (float)pa, nyf = (float)pb, nzf = (float)pc;
    normvec_out = make_float4(nxf, nyf, nzf, pd2);
    // Jacobian row from the stored f32 normal (laserMapping.cpp:1046-1047 reads corr_normvect)
    double n0 = (double)nxf, n1 = (double)nyf, n2 = (double)nzf;
    double pI0 = P.RLI[0] * bx + P.RLI[1] * by + P.RLI[2] * bz + P.TLI[0];
    double pI1 = P.RLI[3] * bx + P.RLI[4] * by + P.RLI[5] * bz + P.TLI[1];
    double pI2 = P.RLI[6] * bx + P.RLI[7] * by + P.RLI[8] * bz + P.TLI[2];
    // C = rot_end^T n
    double C0 = P.R[0] * n0 + P.R[3] * n1 + P.R[6] * n2;
    double C1 = P.R[1] * n0 + P.R[4] * n1 + P.R[7] * n2;
    double C2 = P.R[2] * n0 + P.R[5] * n1 + P.R[8] * n2;
    // A = [pI]x C
    row[0] = pI1 * C2 - pI2 * C1;
    row[1] = pI2 * C0 - pI0 * C2;
    row[2] = pI0 * C1 - pI1 * C0;
    row[3] = n0;
    row[4] = n1;
    row[5] = n2;
    if (IMU) {
        // B = [pL]x (R_LI^T C), C as above (laserMapping.cpp:1057-1059)
        double D0 = P.RLI[0] * C0 + P.RLI[3] * C1 + P.RLI[6] * C2;
        double D1 = P.RLI[1] * C0 + P.RLI[4] * C1 + P.RLI[7] * C2;
        double D2 = P.RLI[2] * C0 + P.RLI[5] * C1 + P.RLI[8] * C2;
        row[6 % L::NC] = by * D2 - bz * D1;
        row[7 % L::NC] = bz * D0 - bx * D2;
        row[8 % L::NC] = bx * D1 - by * D0;
        row[9 % L::NC] = C0;
        row[10 % L::NC] = C1;
        row[11 % L::NC] = C2;
    }
    r = -(double)pd2;   // meas_vec (laserMapping.cpp:1070)
    return true;
}

// Warp reduce-scatter: on entry every lane holds V values; on exit lane l holds the warp sums of
// indices [K*l, K*l+K) in v[0..K). V(1-1/32) shuffles instead of 5V.
template <int N, int S>
struct RS {
    template <int V>
    static __device__ __forceinline__ void run(double (&v)[V], int lane) {
        const bool upper = (lane & S) != 0;
#pragma unroll
        for (int i = 0; i < N; i++) {
            double keep = upper ? v[i + N] : v[i];
            double send = upper ? v[i] : v[i + N];
            v[i] = keep + __shfl_xor_sync(LI_FULL, send, S);
        }
        RS<N / 2, S / 2>::run(v, lane);
    }
};
template <int N>
struct RS<N, 0> {
    template <int V>
    static __device__ __forceinline__ void run(double (&)[V], int) {}
};

// Add one scan point per lane into the warp's accumulators. The V values (upper triangle of row^T row, row*r,
// r^2, 1) are formed and reduce-scattered 32 at a time so that at most 32 doubles are live: afterwards lane l
// holds in acc[g] the running warp sum of value index 32*g + l.
template <bool IMU>
__device__ __forceinline__ void warp_accumulate(const double (&row)[AccLayout<IMU>::NC], double r, bool sel, int lane,
                                                double (&acc)[AccLayout<IMU>::K]) {
    typedef AccLayout<IMU> L;
#pragma unroll
    for (int g = 0; g < L::K; g++) {
        double v[32];
#pragma unroll
        for (int i = 0; i < 32; i++) v[i] = 0.0;
        int idx = 0;
#pragma unroll
        for (int a = 0; a < L::NC; a++) {
#pragma unroll
            for (int b = a; b < L::NC; b++) {
                if (idx / 32 == g) v[idx % 32] = row[a] * row[b];
                idx++;
            }
        }
#pragma unroll
        for (int a = 0; a < L::NC; a++) {
            if (idx / 32 == g) v[idx % 32] = row[a] * r;
            idx++;
        }
        if (idx / 32 == g) v[idx % 32] = r * r;
        idx++;
        if (idx / 32 == g) v[idx % 32] = sel ? 1.0 : 0.0;
        RS<16, 16>::run(v, lane);
        acc[g] += v[0];
    }
}

// ---- multi-GPU: the sum over the ranks INSIDE the reduction's last block, over NVLink peer memory --------------------------
// Every rank owns an exchange buffer [2 phases][nranks][160 doubles] + flags [2][nranks], mapped into every other rank's address
// space (CUDA IPC, liinit_comm_init). The last block of a rank's plane kernel stores its 160-double block into slot `rank` of EVERY
// rank's buffer (peer stores over NVLink), publishes it with a system-scope flag = pass sequence number, waits until all nranks slots
// of its OWN buffer carry that number and sums them in rank order -- the same order on every rank, so all ranks hold bit-identical
// sums (as with ncclAllReduce) and the result does not depend on arrival order. Two phases (seq & 1): a rank can only be one pass ahead
// of the slowest one, because finishing pass s needs everybody's block of pass s.
// No extra launch, no NCCL kernel, no host involvement: the collective costs one NVLink round trip at the tail of the kernel that
// produced its input (SURVEY.md section 8e: "fused at the tail of the kernel").
#define LI_MAX_RANKS 64
struct XchgTable {
    double* blocks[LI_MAX_RANKS];       // rank r's buffer as seen from THIS device
    unsigned* flags[LI_MAX_RANKS];
    double* local;                      // where this rank's own block is kept for liinit_comm_last_local
    int nranks, rank;
};

__device__ __forceinline__ void li_st_release_sys(unsigned* p, unsigned v) {
#ifdef LI_SIMT_EMUL
    *p = v;
#else
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
#endif
}
__device__ __forceinline__ unsigned li_ld_acquire_sys(const unsigned* p) {
#ifdef LI_SIMT_EMUL
    return *p;
#else
    unsigned v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
#endif
}
__device__ __forceinline__ double li_ld_volatile_f64(const double* p) {
#ifdef LI_SIMT_EMUL
    return *p;
#else
    double v;
    asm volatile("ld.volatile.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
    return v;
#endif
}

// Block-level accumulation + deterministic grid reduction.
//   acc[K]: this lane's running sums (value index 32*k + lane). partials: [gridDim.x][V]. out160: final layout
//   [HtH 144 | Htr 12 | res_sq | m | 0 0].
template <bool IMU>
__device__ __forceinline__ void block_finish(const double (&acc)[AccLayout<IMU>::K], double* __restrict__ partials,
                                             unsigned* __restrict__ done_counter, double* __restrict__ out160,
                                             const XchgTable* __restrict__ X = nullptr, unsigned seq = 0u) {
    typedef AccLayout<IMU> L;
    __shared__ double spart[8][L::V];
    __shared__ bool s_last;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nwarps = blockDim.x >> 5;
#pragma unroll
    for (int k = 0; k < L::K; k++) spart[warp][32 * k + lane] = acc[k];
    __syncthreads();
    if (threadIdx.x < L::V) {
        double s = 0;
        for (int w = 0; w < nwarps; w++) s += spart[w][threadIdx.x];
        partials[(size_t)blockIdx.x * L::V + threadIdx.x] = s;
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned ticket = atomicAdd(done_counter, 1u);
        s_last = (ticket == gridDim.x - 1);
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    // last block: every value index is summed over the blocks by one warp -- lane l takes blocks l, l+32, ...
    // (independent loads, pipelined), then a fixed shuffle tree. The order depends only on the grid size, so
    // the result is bit-reproducible run to run.
    __shared__ double s_tot[L::V];
    for (int v = warp; v < L::NV; v += nwarps) {
        double s = 0;
        for (unsigned b = lane; b < gridDim.x; b += 32) s += __ldcg(&partials[(size_t)b * L::V + v]);
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) s += __shfl_xor_sync(LI_FULL, s, o);
        if (lane == 0) s_tot[v] = s;
    }
    __syncthreads();
    __shared__ double s_out[160];
    for (int o = threadIdx.x; o < 160; o += blockDim.x) {
        int src = -1;
        if (o < 144) {
            int a = o / 12, b = o % 12;
            if (a > b) { int tt = a; a = b; b = tt; }
            if (b < L::NC) src = a * L::NC - a * (a - 1) / 2 + (b - a);
        } else if (o < 156) {
            int a = o - 144;
            if (a < L::NC) src = L::NT + a;
        } else if (o == 156) {
            src = L::NT + L::NC;
        } else if (o == 157) {
            src = L::NT + L::NC + 1;
        }
        s_out[o] = (src >= 0) ? s_tot[src] : 0.0;
    }
    __syncthreads();
    if (X == nullptr) {
        for (int o = threadIdx.x; o < 160; o += blockDim.x) out160[o] = s_out[o];
    } else {
        // the one exchange of the path, fused here (see XchgTable)
        const int nr = X->nranks, me = X->rank;
        const int ph = (int)(seq & 1u);
        for (int t = threadIdx.x; t < nr * 160; t += blockDim.x) {
            const int r = t / 160, i = t - r * 160;
            X->blocks[r][(size_t)(ph * nr + me) * 160 + i] = s_out[i];     // peer store (NVLink); r == me: local
        }
        for (int o = threadIdx.x; o < 160; o += blockDim.x) X->local[o] = s_out[o];
        __threadfence_system();
        __syncthreads();
        if ((int)threadIdx.x < nr) li_st_release_sys(X->flags[threadIdx.x] + ph * nr + me, seq);
        if ((int)threadIdx.x < nr) {
            const unsigned* f = X->flags[me] + ph * nr + threadIdx.x;
            while (li_ld_acquire_sys(f) != seq) {
            }
        }
        __syncthreads();
        for (int o = threadIdx.x; o < 160; o += blockDim.x) {
            double s = 0.0;
            for (int r = 0; r < nr; r++) s += li_ld_volatile_f64(X->blocks[me] + (size_t)(ph * nr + r) * 160 + o);   // rank order: identical on every rank
            out160[o] = s;
        }
    }
    if (threadIdx.x == 0) *done_counter = 0u;
}


// Order the 5 neighbours as PointType_CMP does (ikd_Tree.h:57-60): ascending distance, distances closer than
// 1e-10 are ties broken by smaller x. The search already delivers ascending distances, only ties can move.
__device__ __forceinline__ bool tie_order(float4 (&nb)[5], float (&d)[5]) {
    bool moved = false;
#pragma unroll
    for (int pass = 0; pass < 4; pass++) {
#pragma unroll
        for (int k = 0; k < 4 - pass; k++) {
            if (fabsf(d[k] - d[k + 1]) < 1e-10f && nb[k + 1].x < nb[k].x) {
                float4 tq = nb[k]; nb[k] = nb[k + 1]; nb[k + 1] = tq;
                float td = d[k]; d[k] = d[k + 1]; d[k + 1] = td;
                moved = true;
            }
        }
    }
    return moved;
}

// ---- plane / residual / Jacobian / reduction pass -----------------------------------------------------
// The pass works on S.near_xyz, the device copy of Nearest_Points (laserMapping.cpp:107): five float4 per scan point, w = 1
// for a neighbour that exists, 0 for a missing rank. They are COPIES of the map points, as in the reference, so reuse passes and
// map_incremental keep working on them whatever happens to the map in between (Add_Points, box deletes, slab moves).
// SEARCH = true : runs right after the search kernel of the same pass; the selection gate is "5 neighbours found"
//                 (laserMapping.cpp:981-984; d2[4] <= 5 holds by construction of the search).
//                 FROM_IDS = true : the search kernel left pool offsets in S.near_ids (lockstep / cell-directory searches): gather
//                                   them here and write S.near_xyz;
//                 FROM_IDS = false: the search kernel wrote S.near_xyz itself (knn_wq.cuh).
//                 Either way the PointType_CMP tie order is applied here and S.near_xyz holds the ordered neighbours afterwards.
// SEARCH = false: reuse pass (nearest_search_en == false, :989-994): previous flag and stored neighbours.
template <bool IMU, bool SEARCH, bool FROM_IDS>
__global__ void __launch_bounds__(256, LI_PLANE_MIN_BLOCKS) k_icp_plane(MapDev M, ScanDev S, PoseD P, double* __restrict__ partials,
                                                   unsigned* __restrict__ done_counter, double* __restrict__ out160,
                                                   const XchgTable* __restrict__ X, unsigned seq) {
    typedef AccLayout<IMU> L;
    const int lane = threadIdx.x & 31;
    double acc[L::K];
#pragma unroll
    for (int k = 0; k < L::K; k++) acc[k] = 0.0;
    const int stride = gridDim.x * blockDim.x;
    const int nround = (S.n + stride - 1) / stride;
    for (int it = 0; it < nround; it++) {
        const int q = it * stride + blockIdx.x * blockDim.x + threadIdx.x;
        double row[L::NC];
        double r = 0.0;
        bool sel = false;
#pragma unroll
        for (int i = 0; i < L::NC; i++) row[i] = 0.0;
        if (q < S.n) {
            const float4 b = __ldg(&S.body[q]);
            const bool gate = SEARCH ? true : (S.selected[q] != 0);
            float4 nb[5];
            if (SEARCH && FROM_IDS) {
                int id[5];
#pragma unroll
                for (int k = 0; k < 5; k++) id[k] = S.near_ids[(size_t)q * 5 + k];
#pragma unroll
                for (int k = 0; k < 5; k++) {
                    nb[k] = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (id[k] >= 0) {
                        nb[k] = __ldg(&M.pool[id[k]]);
                        nb[k].w = 1.0f;
                    }
                }
            } else {
#pragma unroll
                for (int k = 0; k < 5; k++) nb[k] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (gate) {
#pragma unroll
                    for (int k = 0; k < 5; k++) nb[k] = S.near_xyz[(size_t)q * 5 + k];
                }
            }
            float wx, wy, wz;
            li_body_to_world(P, b.x, b.y, b.z, wx, wy, wz);
            if (!SEARCH) S.world[q] = make_float4(wx, wy, wz, 0.f);
            const bool fit = gate && nb[4].w != 0.f;
            if (SEARCH) {
                // the ordered copies are stored before the plane fit, so that nothing but the fit's own inputs is live across the QR
                bool moved = false;
                if (fit) {
                    float d[5];
#pragma unroll
                    for (int k = 0; k < 5; k++) d[k] = li_dist2(wx, wy, wz, nb[k].x, nb[k].y, nb[k].z);
                    moved = tie_order(nb, d);
                }
                if (FROM_IDS || moved) {
#pragma unroll
                    for (int k = 0; k < 5; k++) S.near_xyz[(size_t)q * 5 + k] = nb[k];
                }
            }
            if (fit) {
                float4 nvec;
                sel = plane_and_row<IMU>(P, b.x, b.y, b.z, wx, wy, wz, nb, nvec, row, r);
                if (sel) S.normvec[q] = nvec;
            }
            S.selected[q] = sel ? 1 : 0;
        }
        warp_accumulate<IMU>(row, r, sel, lane, acc);
    }
    block_finish<IMU>(acc, partials, done_counter, out160, X, seq);
}
