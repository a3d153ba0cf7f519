// assess_time_kernels.cuh -- the timed map assessment (liinit_assess_*_timed, DESIGN.md section 4d): every evaluation re-undistorts the
// raw points of the timed scans for its candidate extrinsic and lag shift before it places them.
//
// A timed scan keeps its raw points (xyz, w = time [ms]), the IMU pose table liinit_raw_undistort_imu got and the propagated state of
// that call. A lag shift delta [s] moves the candidate's pose table: its value at time u is the run's at u + delta. So a point at tau
// [ms] is undistorted at t = tau / 1000 + delta in the run's table, towards the scan-end state carried delta further with the table's
// last gyro and acceleration (the reference's own end-of-frame extrapolation, IMU_Processing.hpp:374-378). At delta = 0 and the prior
// extrinsic this is k_undistort_imu's arithmetic on the same operands (li_undistort_imu_point), so the placement is bit-equal to the
// plain store's. Untimed scans are placed from their stored (undistorted) points exactly as k_as_place does.
#pragma once
#include "common.cuh"
#include "undistort_kernels.cuh"
#include "assess_kernels.cuh"

// per stored scan of a timed store: the pose table (rows [row0, row0 + npose) of the pool; npose = 0: an untimed scan) and the state
// passed to liinit_raw_undistort_imu (rot_end, pos_end, R_LI, T_LI; vel_end)
struct AtScan {
    PoseD prior;
    double vel[3];
    long long row0;
    int npose;
    int pad;
};

// the undistortion target of every timed scan for lag shift delta: R_e = R_prop Exp(gyr_last, delta), p_e = p_prop + v_prop delta +
// 1/2 acc_last delta^2 (delta = 0: the prior as it is), with the candidate extrinsic (as_run: the prior's)
__global__ void k_at_scan_end(const AtScan* __restrict__ at, const double* __restrict__ pool, int scans, double delta, int as_run, PoseD cand,
                              PoseD* __restrict__ end) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= scans) return;
    const AtScan& A = at[s];
    PoseD E = as_run ? A.prior : cand;
#pragma unroll
    for (int k = 0; k < 9; k++) E.R[k] = A.prior.R[k];
#pragma unroll
    for (int k = 0; k < 3; k++) E.p[k] = A.prior.p[k];
    if (A.npose >= 2 && delta != 0.0) {
        const double* last = pool + (size_t)(A.row0 + A.npose - 1) * LI_POSE6D_DOUBLES;
        double X[9];
        li_so3_exp_dt(last + 4, delta, X);
        const double* Rp = A.prior.R;
#pragma unroll
        for (int a = 0; a < 3; a++)
#pragma unroll
            for (int b = 0; b < 3; b++) E.R[3 * a + b] = Rp[3 * a] * X[b] + Rp[3 * a + 1] * X[3 + b] + Rp[3 * a + 2] * X[6 + b];
#pragma unroll
        for (int a = 0; a < 3; a++) E.p[a] = A.prior.p[a] + A.vel[a] * delta + 0.5 * last[1 + a] * delta * delta;
    }
    end[s] = E;
}

// place, timed: a point of a timed scan is undistorted from its raw copy at t = tau / 1000 + delta (head row as k_undistort_imu; no
// head: untouched at delta = 0, row 0 with dt < 0 otherwise) towards end[scan], then placed like k_as_place; untimed points as
// k_as_place. The cell box as li_as_box.
__global__ void k_at_place(const float4* __restrict__ pts, const float4* __restrict__ raw, const PoseD* __restrict__ poses,
                           const AtScan* __restrict__ at, const PoseD* __restrict__ end, const double* __restrict__ pool, int n, double delta,
                           int as_run, PoseD cand, double edge, float4* __restrict__ world, int* __restrict__ box) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    int c[3] = {0x7fffffff, 0x7fffffff, 0x7fffffff}, C[3] = {-0x7fffffff - 1, -0x7fffffff - 1, -0x7fffffff - 1};
    int bad = 0;
    if (i < n) {
        const float4 p = pts[i];
        const int s = __float_as_int(p.w);
        float x = p.x, y = p.y, z = p.z;
        const int npose = at[s].npose;
        if (npose >= 2) {
            const float4 r = raw[i];
            const double t0 = (double)r.w / 1000.0;
            const double t = delta != 0.0 ? t0 + delta : t0;
            const double* tab = pool + (size_t)at[s].row0 * LI_POSE6D_DOUBLES;
            int head = li_imu_head(tab, npose, t);
            if (head < 0 && delta != 0.0) head = 0;
            x = r.x; y = r.y; z = r.z;
            if (head >= 0) {
                const float3 u = li_undistort_imu_point(tab + (size_t)head * LI_POSE6D_DOUBLES, t, end[s], r.x, r.y, r.z);
                x = u.x; y = u.y; z = u.z;
            }
        }
        const PoseD P = li_as_pose(poses[s], as_run, cand);
        float w[3];
        li_body_to_world(P, x, y, z, w[0], w[1], w[2]);
        world[i] = make_float4(w[0], w[1], w[2], 0.f);
        li_as_cells(w, edge, c, C, bad);
    }
    li_as_box(c, C, bad, box);
}
