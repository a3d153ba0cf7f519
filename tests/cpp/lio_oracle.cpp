// tests/cpp/lio_oracle.cpp -- TEST INFRASTRUCTURE ONLY: the CPU checker of the LIO mode, next to oracle/ (which it does not change).
//
// Restated on its own from the reference, sharing no code with lidar_imu_init_b200/csrc/host/liinit_host.cpp:
//   * the forward part of ImuProcess::propagation_and_undist (src/IMU_Processing.hpp:269-382), literally: dense F, dense cov_w,
//     two dense products;
//   * pointBodyToWorld (src/laserMapping.cpp:209-220): double math, float store.
// Built on demand by tests/lio_oracle.py (g++ -O3 -std=c++14 -ffp-contract=off, the flags of oracle/Makefile).
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <vector>

namespace {

// StatesGroup (common_lib.h:68-169), flat: the layout of struct liinit_state and of oracle/liinit_oracle.cpp's State.
struct State {
    double rot_end[9], pos_end[3], R_LI[9], T_LI[3], vel[3], bg[3], ba[3], grav[3];
    double cov[24 * 24];
};

void mat3_mul_vec(const double* R, const double* v, double* o) {   // row-major 3x3
    for (int i = 0; i < 3; i++) o[i] = R[3 * i] * v[0] + R[3 * i + 1] * v[1] + R[3 * i + 2] * v[2];
}
void mat3_mul(const double* A, const double* B, double* C) {
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
void skew(const double* v, double* K) {   // so3_math.h:8
    K[0] = 0; K[1] = -v[2]; K[2] = v[1];
    K[3] = v[2]; K[4] = 0; K[5] = -v[0];
    K[6] = -v[1]; K[7] = v[0]; K[8] = 0;
}
// Exp(ang_vel, dt) (so3_math.h:39-59)
void so3_exp_dt(const double* w, double dt, double* R) {
    const double n = std::sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
    const double I[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    if (n > 0.0000001) {
        double r[3] = {w[0] / n, w[1] / n, w[2] / n};
        double K[9], KK[9];
        skew(r, K);
        mat3_mul(K, K, KK);
        const double a = n * dt, s = std::sin(a), c = 1.0 - std::cos(a);
        for (int i = 0; i < 9; i++) R[i] = I[i] + s * K[i] + c * KK[i];
    } else {
        for (int i = 0; i < 9; i++) R[i] = I[i];
    }
}

}  // namespace

extern "C" {

int lio_oracle_state_doubles() { return (int)(sizeof(State) / sizeof(double)); }

// The forward part of propagation_and_undist (IMU_Processing.hpp:269-382), literal: dense 24x24 F and cov_w, cov = F cov F^T + cov_w
// as two dense products. imu: the ImuProcess members, flat, 33 doubles:
//   last_imu_ {stamp, gyr[3], acc[3]} 0:7 | angvel_last 7:10 | acc_s_last 10:13 | last_lidar_end_time_ 13 | cov_acc 14:17 |
//   cov_gyr 17:20 | cov_R_LI 20:23 | cov_T_LI 23:26 | cov_bias_gyr 26:29 | cov_bias_acc 29:32 | IMU_mean_acc_norm 32,
// updated in place like the members. samples: n x {stamp, gyr[3], acc[3]}. state: struct State, in/out.
// poses: room for n + 1 Pose6D (22 doubles). Returns the number of poses (IMUpose.size()).
int lio_oracle_propagate_imu(double* imu, double* state, const double* samples, int n, double pcl_beg_time, double pcl_end_offset_ms,
                         double* poses) {
    if (n <= 0) return 0;   // Process returns on an empty group (IMU_Processing.hpp:423)
    struct Smp { double t, g[3], a[3]; };
    auto rd = [](const double* p) { Smp s; s.t = p[0]; for (int i = 0; i < 3; i++) { s.g[i] = p[1 + i]; s.a[i] = p[4 + i]; } return s; };
    State& st = *reinterpret_cast<State*>(state);
    double* angvel_last = imu + 7;
    double* acc_s_last = imu + 10;
    double& last_lidar_end_time_ = imu[13];
    const double *cov_acc = imu + 14, *cov_gyr = imu + 17, *cov_R_LI = imu + 20, *cov_T_LI = imu + 23, *cov_bias_gyr = imu + 26,
                 *cov_bias_acc = imu + 29;
    const double IMU_mean_acc_norm = imu[32];
    const double G_m_s2 = 9.81;
    std::vector<Smp> v_imu;
    v_imu.push_back(rd(imu));                                     // v_imu.push_front(last_imu_)
    for (int k = 0; k < n; k++) v_imu.push_back(rd(samples + 7 * (size_t)k));
    const double imu_end_time = v_imu.back().t;
    const double pcl_end_time = pcl_beg_time + pcl_end_offset_ms / double(1000);
    int np = 0;
    auto push_pose = [&](double t, const double* a, const double* g, const double* v, const double* p, const double* R) {
        double* o = poses + 22 * (size_t)np++;
        o[0] = t;
        for (int i = 0; i < 3; i++) { o[1 + i] = a[i]; o[4 + i] = g[i]; o[7 + i] = v[i]; o[10 + i] = p[i]; }
        for (int i = 0; i < 9; i++) o[13 + i] = R[i];
    };
    push_pose(0.0, acc_s_last, angvel_last, st.vel, st.pos_end, st.rot_end);
    double acc_imu[3] = {0, 0, 0}, angvel_avr[3] = {0, 0, 0}, acc_avr[3], vel_imu[3], pos_imu[3], R_imu[9];
    for (int i = 0; i < 3; i++) { vel_imu[i] = st.vel[i]; pos_imu[i] = st.pos_end[i]; }
    for (int i = 0; i < 9; i++) R_imu[i] = st.rot_end[i];
    static thread_local double F[24 * 24], Q[24 * 24], FP[24 * 24];
    double dt = 0;
    for (size_t it = 0; it + 1 < v_imu.size(); it++) {
        const Smp& head = v_imu[it];
        const Smp& tail = v_imu[it + 1];
        if (tail.t < last_lidar_end_time_) continue;
        for (int i = 0; i < 3; i++) {
            angvel_avr[i] = 0.5 * (head.g[i] + tail.g[i]);
            acc_avr[i] = 0.5 * (head.a[i] + tail.a[i]);
        }
        for (int i = 0; i < 3; i++) {
            angvel_avr[i] -= st.bg[i];
            acc_avr[i] = acc_avr[i] / IMU_mean_acc_norm * G_m_s2 - st.ba[i];
        }
        if (head.t < last_lidar_end_time_) dt = tail.t - last_lidar_end_time_;
        else dt = tail.t - head.t;
        double Exp_f[9], Exp_b[9], K[9], RK[9];
        so3_exp_dt(angvel_avr, dt, Exp_f);
        so3_exp_dt(angvel_avr, -dt, Exp_b);
        skew(acc_avr, K);
        mat3_mul(R_imu, K, RK);
        std::fill(F, F + 576, 0.0);
        std::fill(Q, Q + 576, 0.0);
        for (int i = 0; i < 24; i++) F[i * 24 + i] = 1.0;
        for (int i = 0; i < 3; i++) {
            for (int j = 0; j < 3; j++) {
                F[i * 24 + j] = Exp_b[3 * i + j];                        // F(0:3, 0:3)
                F[(12 + i) * 24 + j] = -RK[3 * i + j] * dt;              // F(12:15, 0:3)
                F[(12 + i) * 24 + 18 + j] = -R_imu[3 * i + j] * dt;      // F(12:15, 18:21)
            }
            F[i * 24 + 15 + i] = -dt;                                    // F(0:3, 15:18)
            F[(3 + i) * 24 + 12 + i] = dt;                               // F(3:6, 12:15)
            F[(12 + i) * 24 + 21 + i] = dt;                              // F(12:15, 21:24)
            Q[i * 24 + i] = cov_gyr[i] * dt * dt;
            Q[(6 + i) * 24 + 6 + i] = cov_R_LI[i] * dt * dt;
            Q[(9 + i) * 24 + 9 + i] = cov_T_LI[i] * dt * dt;
            Q[(15 + i) * 24 + 15 + i] = cov_bias_gyr[i] * dt * dt;
            Q[(18 + i) * 24 + 18 + i] = cov_bias_acc[i] * dt * dt;
            for (int j = 0; j < 3; j++) {                                // R_imu * cov_acc.asDiagonal() * R_imu^T
                double s = 0;
                for (int k = 0; k < 3; k++) s += R_imu[3 * i + k] * cov_acc[k] * R_imu[3 * j + k];
                Q[(12 + i) * 24 + 12 + j] = s * dt * dt;
            }
        }
        for (int r = 0; r < 24; r++)
            for (int c = 0; c < 24; c++) {
                double s = 0;
                for (int k = 0; k < 24; k++) s += F[r * 24 + k] * st.cov[k * 24 + c];
                FP[r * 24 + c] = s;
            }
        for (int r = 0; r < 24; r++)
            for (int c = 0; c < 24; c++) {
                double s = 0;
                for (int k = 0; k < 24; k++) s += FP[r * 24 + k] * F[c * 24 + k];
                st.cov[r * 24 + c] = s + Q[r * 24 + c];
            }
        double Rn[9];
        mat3_mul(R_imu, Exp_f, Rn);
        for (int i = 0; i < 9; i++) R_imu[i] = Rn[i];
        mat3_mul_vec(R_imu, acc_avr, acc_imu);
        for (int i = 0; i < 3; i++) acc_imu[i] += st.grav[i];
        for (int i = 0; i < 3; i++) {
            pos_imu[i] = pos_imu[i] + vel_imu[i] * dt + 0.5 * acc_imu[i] * dt * dt;
            vel_imu[i] = vel_imu[i] + acc_imu[i] * dt;
        }
        for (int i = 0; i < 3; i++) { angvel_last[i] = angvel_avr[i]; acc_s_last[i] = acc_imu[i]; }
        push_pose(tail.t - pcl_beg_time, acc_imu, angvel_avr, vel_imu, pos_imu, R_imu);
    }
    const double note = pcl_end_time > imu_end_time ? 1.0 : -1.0;
    dt = note * (pcl_end_time - imu_end_time);
    double w[3] = {note * angvel_avr[0], note * angvel_avr[1], note * angvel_avr[2]}, E[9];
    so3_exp_dt(w, dt, E);
    mat3_mul(R_imu, E, st.rot_end);
    for (int i = 0; i < 3; i++) {
        st.vel[i] = vel_imu[i] + note * acc_imu[i] * dt;
        st.pos_end[i] = pos_imu[i] + note * vel_imu[i] * dt + note * 0.5 * acc_imu[i] * dt * dt;
    }
    for (int i = 0; i < 7; i++) imu[i] = samples[7 * (size_t)(n - 1) + i];   // last_imu_ = meas.imu.back()
    last_lidar_end_time_ = pcl_end_time;
    return np;
}

// pointBodyToWorld (laserMapping.cpp:209-220) over n points: xyz [n*3] body -> out [n*3] world.
void lio_oracle_body_to_world(const float* xyz, int n, const double* rot_end, const double* pos_end, const double* R_LI, const double* T_LI,
                          float* out) {
    for (int i = 0; i < n; i++) {
        const double pb[3] = {xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2]};
        double t[3], g[3];
        mat3_mul_vec(R_LI, pb, t);
        for (int a = 0; a < 3; a++) t[a] += T_LI[a];
        mat3_mul_vec(rot_end, t, g);
        for (int a = 0; a < 3; a++) out[3 * (size_t)i + a] = (float)(g[a] + pos_end[a]);
    }
}

}  // extern "C"
