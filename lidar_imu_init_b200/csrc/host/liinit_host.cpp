// liinit_host.cpp -- host side of the drop-in (see liinit_host.h). Everything here is O(24^3) per iteration.
#include "liinit_host.h"

#include <array>
#include <cmath>
#include <cstring>
#include <deque>
#include <vector>

namespace {

constexpr int D = LIINIT_DIM_STATE;

inline void mul33(const double* A, const double* B, double* C) {
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
inline void mulT33(const double* A, const double* B, double* C) {   // A^T * B
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) C[3 * i + j] = A[i] * B[j] + A[3 + i] * B[3 + j] + A[6 + i] * B[6 + j];
}

// Dense inverse by LU with partial pivoting (what Eigen's .inverse() does for a 24x24, laserMapping.cpp:1081).
// ncols < n: only the first ncols columns of the inverse are solved for (the others of X are left untouched) -- the gain K_1 enters
// the update through its first 12 columns only; a column of the inverse does not depend on which other columns are computed.
bool invert(const double* A, double* X, int n, int ncols = -1) {
    if (ncols < 0) ncols = n;
    double lu[D * D];
    int perm[D];
    std::memcpy(lu, A, sizeof(double) * n * n);
    for (int i = 0; i < n; i++) perm[i] = i;
    for (int k = 0; k < n; k++) {
        int piv = k;
        double best = std::fabs(lu[k * n + k]);
        for (int i = k + 1; i < n; i++)
            if (std::fabs(lu[i * n + k]) > best) {
                best = std::fabs(lu[i * n + k]);
                piv = i;
            }
        if (best == 0.0) return false;
        if (piv != k) {
            for (int j = 0; j < n; j++) {
                double t = lu[k * n + j];
                lu[k * n + j] = lu[piv * n + j];
                lu[piv * n + j] = t;
            }
            int t = perm[k];
            perm[k] = perm[piv];
            perm[piv] = t;
        }
        const double inv = 1.0 / lu[k * n + k];
        for (int i = k + 1; i < n; i++) {
            const double f = lu[i * n + k] * inv;
            lu[i * n + k] = f;
            for (int j = k + 1; j < n; j++) lu[i * n + j] -= f * lu[k * n + j];
        }
    }
    for (int c = 0; c < ncols; c++) {
        double y[D];
        for (int i = 0; i < n; i++) {
            double s = (perm[i] == c) ? 1.0 : 0.0;
            for (int j = 0; j < i; j++) s -= lu[i * n + j] * y[j];
            y[i] = s;
        }
        for (int i = n - 1; i >= 0; i--) {
            double s = y[i];
            for (int j = i + 1; j < n; j++) s -= lu[i * n + j] * X[j * n + c];
            X[i * n + c] = s / lu[i * n + i];
        }
    }
    return true;
}

}  // namespace

extern "C" {

void liinit_so3_exp(const double v[3], double R[9]) {
    const double n = std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    static const double I[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    if (n > 0.00001) {   // so3_math.h:66
        const double r[3] = {v[0] / n, v[1] / n, v[2] / n};
        const double K[9] = {0, -r[2], r[1], r[2], 0, -r[0], -r[1], r[0], 0};
        double KK[9];
        mul33(K, K, KK);
        const double s = std::sin(n), c = 1.0 - std::cos(n);
        for (int i = 0; i < 9; i++) R[i] = I[i] + s * K[i] + c * KK[i];
    } else {
        std::memcpy(R, I, sizeof(I));
    }
}

void liinit_so3_log(const double R[9], double v[3]) {
    const double tr = R[0] + R[4] + R[8];
    const double theta = (tr > 3.0 - 1e-6) ? 0.0 : std::acos(0.5 * (tr - 1));
    const double f = (std::fabs(theta) < 0.001) ? 0.5 : (0.5 * theta / std::sin(theta));
    v[0] = f * (R[7] - R[5]);
    v[1] = f * (R[2] - R[6]);
    v[2] = f * (R[3] - R[1]);
}

void liinit_state_init(liinit_state* s) {
    std::memset(s, 0, sizeof(*s));
    s->rot_end[0] = s->rot_end[4] = s->rot_end[8] = 1.0;
    s->offset_R_L_I[0] = s->offset_R_L_I[4] = s->offset_R_L_I[8] = 1.0;
    for (int i = 0; i < D; i++) s->cov[i * D + i] = (i >= 15) ? 0.00001 : 1.0;   // INIT_COV, common_lib.h:79-80
}

void liinit_state_boxplus(liinit_state* s, const double* d) {
    double E[9], R[9];
    liinit_so3_exp(d, E);
    mul33(s->rot_end, E, R);
    std::memcpy(s->rot_end, R, sizeof(R));
    liinit_so3_exp(d + 6, E);
    mul33(s->offset_R_L_I, E, R);
    std::memcpy(s->offset_R_L_I, R, sizeof(R));
    for (int i = 0; i < 3; i++) {
        s->pos_end[i] += d[3 + i];
        s->offset_T_L_I[i] += d[9 + i];
        s->vel_end[i] += d[12 + i];
        s->bias_g[i] += d[15 + i];
        s->bias_a[i] += d[18 + i];
        s->gravity[i] += d[21 + i];
    }
}

void liinit_state_boxminus(const liinit_state* a, const liinit_state* b, double* o) {
    double rd[9];
    mulT33(b->rot_end, a->rot_end, rd);
    liinit_so3_log(rd, o);
    mulT33(b->offset_R_L_I, a->offset_R_L_I, rd);
    liinit_so3_log(rd, o + 6);
    for (int i = 0; i < 3; i++) {
        o[3 + i] = a->pos_end[i] - b->pos_end[i];
        o[9 + i] = a->offset_T_L_I[i] - b->offset_T_L_I[i];
        o[12 + i] = a->vel_end[i] - b->vel_end[i];
        o[15 + i] = a->bias_g[i] - b->bias_g[i];
        o[18 + i] = a->bias_a[i] - b->bias_a[i];
        o[21 + i] = a->gravity[i] - b->gravity[i];
    }
}

// cov_inv: state.cov^-1 when the caller already has it (the covariance does not change between the iterations of a scan,
// laserMapping.cpp:1081 vs :1127: liinit_scan_update inverts it once), else nullptr.
static int ieskf_update(liinit_state* st, const liinit_state* prop, const double* HtH, const double* Htr, double* sol, double* KH,
                        const double* cov_inv) {
    double S[D * D], K1[D * D];
    if (cov_inv) std::memcpy(S, cov_inv, sizeof(S));
    else if (!invert(st->cov, S, D)) return LIINIT_ERR_INVALID;      // cov^-1
    for (int a = 0; a < 12; a++)
        for (int b = 0; b < 12; b++) S[a * D + b] += 1000.0 * HtH[a * 12 + b];   // R_inv = 1000 (laserMapping.cpp:1050)
    if (!invert(S, K1, D, 12)) return LIINIT_ERR_INVALID;            // (columns 0..11 of K_1 are all the update reads)
    double vec[D];
    liinit_state_boxminus(prop, st, vec);
    double G[D * 12];   // K*Hsub
    for (int r = 0; r < D; r++)
        for (int c = 0; c < 12; c++) {
            double s = 0;
            for (int a = 0; a < 12; a++) s += K1[r * D + a] * (1000.0 * HtH[a * 12 + c]);
            G[r * 12 + c] = s;
        }
    for (int r = 0; r < D; r++) {
        double s = 0, t = 0;
        for (int a = 0; a < 12; a++) {
            s += K1[r * D + a] * (1000.0 * Htr[a]);
            t += G[r * 12 + a] * vec[a];
        }
        sol[r] = s + vec[r] - t;
    }
    liinit_state_boxplus(st, sol);
    if (KH) std::memcpy(KH, G, sizeof(G));
    return LIINIT_OK;
}

int liinit_ieskf_update(liinit_state* st, const liinit_state* prop, const double* HtH, const double* Htr, double* sol, double* KH) {
    return ieskf_update(st, prop, HtH, Htr, sol, KH, nullptr);
}

// ---- the update with a constant extrinsic: the 18 states other than R_LI (6:9) and T_LI (9:12) ----
constexpr int DF = D - 6;
static const int kFree[DF] = {0, 1, 2, 3, 4, 5, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23};

// cov restricted to the free states, inverted (DF x DF)
static bool free_cov_inverse(const double* P, double* out) {
    double Pr[DF * DF];
    for (int r = 0; r < DF; r++)
        for (int c = 0; c < DF; c++) Pr[r * DF + c] = P[kFree[r] * D + kFree[c]];
    return invert(Pr, out, DF);
}

static void zero_extrinsic_cov(double* P) {
    for (int i = 6; i < 12; i++)
        for (int j = 0; j < D; j++) P[i * D + j] = P[j * D + i] = 0.0;
}

// ieskf_update on the free states: K_1 = (blkdiag(1000 HtH[0:6,0:6], 0) + cov_r^-1)^-1, solution_r = K_1[:,0:6] (1000 Htr[0:6]) + vec_r -
// K_1[:,0:6] (1000 HtH[0:6,0:6]) vec[0:6]; the extrinsic keeps its bits (Exp(0) and + 0 could still flip the sign of a zero)
static int ieskf_update_frozen(liinit_state* st, const liinit_state* prop, const double* HtH, const double* Htr, double* sol, double* KH,
                               const double* cov_inv_r) {
    double S[DF * DF], K1[DF * DF];
    if (cov_inv_r) std::memcpy(S, cov_inv_r, sizeof(S));
    else if (!free_cov_inverse(st->cov, S)) return LIINIT_ERR_INVALID;
    for (int a = 0; a < 6; a++)
        for (int b = 0; b < 6; b++) S[a * DF + b] += 1000.0 * HtH[a * 12 + b];
    if (!invert(S, K1, DF, 6)) return LIINIT_ERR_INVALID;
    double vec[D], vr[DF];
    liinit_state_boxminus(prop, st, vec);
    for (int i = 0; i < DF; i++) vr[i] = vec[kFree[i]];
    double G[DF * 6];
    for (int r = 0; r < DF; r++)
        for (int c = 0; c < 6; c++) {
            double s = 0;
            for (int a = 0; a < 6; a++) s += K1[r * DF + a] * (1000.0 * HtH[a * 12 + c]);
            G[r * 6 + c] = s;
        }
    for (int i = 0; i < D; i++) sol[i] = 0.0;
    for (int r = 0; r < DF; r++) {
        double s = 0, t = 0;
        for (int a = 0; a < 6; a++) {
            s += K1[r * DF + a] * (1000.0 * Htr[a]);
            t += G[r * 6 + a] * vr[a];
        }
        sol[kFree[r]] = s + vr[r] - t;
    }
    double RLI[9], TLI[3];
    std::memcpy(RLI, st->offset_R_L_I, sizeof(RLI));
    std::memcpy(TLI, st->offset_T_L_I, sizeof(TLI));
    liinit_state_boxplus(st, sol);
    std::memcpy(st->offset_R_L_I, RLI, sizeof(RLI));
    std::memcpy(st->offset_T_L_I, TLI, sizeof(TLI));
    if (KH) {
        for (int i = 0; i < D * 12; i++) KH[i] = 0.0;
        for (int r = 0; r < DF; r++)
            for (int c = 0; c < 6; c++) KH[kFree[r] * 12 + c] = G[r * 6 + c];
    }
    zero_extrinsic_cov(st->cov);
    return LIINIT_OK;
}

int liinit_ieskf_update_frozen(liinit_state* st, const liinit_state* prop, const double* HtH, const double* Htr, double* sol, double* KH) {
    return ieskf_update_frozen(st, prop, HtH, Htr, sol, KH, nullptr);
}

static int scan_update(liinit_ctx* h, liinit_state* state, int max_iter, int imu_en, liinit_scan_stats* stats, bool frozen) {
    if (!h || !state || max_iter < 1) return LIINIT_ERR_INVALID;
    liinit_state prop = *state;            // state_propagat = state (laserMapping.cpp:910)
    int rematch_num = 0, nearest_search_en = 1;
    liinit_scan_stats st{};
    double HtH[144], Htr[12], sol[D], KH[D * 12];
    double cov_inv[D * D];                 // state.cov is only replaced at the end of the scan (:1127): one inversion for all iterations
    if (!(frozen ? free_cov_inverse(state->cov, cov_inv) : invert(state->cov, cov_inv, D))) return LIINIT_ERR_INVALID;
    if (frozen) zero_extrinsic_cov(state->cov);
    for (int it = 0; it < max_iter; it++) {
        int m = 0;
        double rs = 0;
        st.search_passes += nearest_search_en;
        int rc = liinit_icp_iterate(h, state->rot_end, state->pos_end, state->offset_R_L_I, state->offset_T_L_I, imu_en,
                                    nearest_search_en, HtH, Htr, &m, &rs);
        if (rc != LIINIT_OK) return rc;
        rc = frozen ? ieskf_update_frozen(state, &prop, HtH, Htr, sol, KH, cov_inv) : ieskf_update(state, &prop, HtH, Htr, sol, KH, cov_inv);
        if (rc != LIINIT_OK) return rc;
        st.iterations++;
        st.effect_feat_num = m;
        st.res_sq = rs;
        const double rn = std::sqrt(sol[0] * sol[0] + sol[1] * sol[1] + sol[2] * sol[2]);
        const double tn = std::sqrt(sol[3] * sol[3] + sol[4] * sol[4] + sol[5] * sol[5]);
        st.last_rot_deg = rn * 57.3;
        st.last_trans_cm = tn * 100;
        const bool converged = (rn * 57.3 < 0.01) && (tn * 100 < 0.015);       // :1093-1094
        st.converged = converged;
        nearest_search_en = 0;                                                 // :1102-1106
        if (converged || (rematch_num == 0 && it == max_iter - 2)) {
            nearest_search_en = 1;
            rematch_num++;
        }
        if (rematch_num >= 2 || it == max_iter - 1) {                          // :1109-1133
            double nc[D * D];
            for (int r = 0; r < D; r++)
                for (int c = 0; c < D; c++) {
                    double s = state->cov[r * D + c];
                    for (int a = 0; a < 12; a++) s -= KH[r * 12 + a] * state->cov[a * D + c];
                    nc[r * D + c] = s;
                }
            std::memcpy(state->cov, nc, sizeof(nc));
            break;
        }
    }
    if (stats) *stats = st;
    return LIINIT_OK;
}

int liinit_scan_update(liinit_ctx* h, liinit_state* state, int max_iter, int imu_en, liinit_scan_stats* stats) {
    return scan_update(h, state, max_iter, imu_en, stats, false);
}

int liinit_scan_update_frozen(liinit_ctx* h, liinit_state* state, int max_iter, int imu_en, liinit_scan_stats* stats) {
    return scan_update(h, state, max_iter, imu_en, stats, true);
}

// Exp(ang_vel, dt) (so3_math.h:39-59): gated on the angular VELOCITY (|w| > 1e-7), not on the angle like Exp(v1, v2, v3) (:61-80,
// |v| > 1e-5) -- for 1e-7 < |w| < 1e-5 / dt the two differ (identity vs a small rotation). The un-distortion kernel uses the same
// form (li_so3_exp_dt, undistort_kernels.cuh).
static void so3_exp_dt(const double w[3], double dt, double R[9]) {
    const double n = std::sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
    for (int i = 0; i < 9; i++) R[i] = (i % 4 == 0) ? 1.0 : 0.0;
    if (!(n > 0.0000001)) return;
    const double a[3] = {w[0] / n, w[1] / n, w[2] / n};
    const double K[9] = {0, -a[2], a[1], a[2], 0, -a[0], -a[1], a[0], 0};
    double KK[9];
    mul33(K, K, KK);
    const double ang = n * dt, sn = std::sin(ang), cs = 1.0 - std::cos(ang);
    for (int i = 0; i < 9; i++) R[i] += sn * K[i] + cs * KK[i];
}

void liinit_propagate_cv(liinit_state* s, double dt, const double* cov_gyr_scale, const double* cov_acc_scale) {
    // F is the identity except three 3x3 blocks, so F cov F^T touches rows / columns 0:6 only:
    //   rows 0:3 <- E rows 0:3 + dt rows 15:18 ; rows 3:6 <- rows 3:6 + dt rows 12:15 ; then the same on the columns.
    double E[9];
    so3_exp_dt(s->bias_g, -dt, E);   // Exp(state_inout.bias_g, -dt) (IMU_Processing.hpp:226)
    std::vector<double> T(D * D);
    double* P = s->cov;
    for (int c = 0; c < D; c++) {
        for (int r = 0; r < D; r++) T[r * D + c] = P[r * D + c];
        for (int r = 0; r < 3; r++)
            T[r * D + c] = E[3 * r] * P[0 * D + c] + E[3 * r + 1] * P[1 * D + c] + E[3 * r + 2] * P[2 * D + c] + dt * P[(15 + r) * D + c];
        for (int r = 0; r < 3; r++) T[(3 + r) * D + c] = P[(3 + r) * D + c] + dt * P[(12 + r) * D + c];
    }
    for (int r = 0; r < D; r++) {
        for (int c = 0; c < D; c++) P[r * D + c] = T[r * D + c];
        for (int c = 0; c < 3; c++)
            P[r * D + c] = T[r * D + 0] * E[3 * c] + T[r * D + 1] * E[3 * c + 1] + T[r * D + 2] * E[3 * c + 2] + dt * T[r * D + 15 + c];
        for (int c = 0; c < 3; c++) P[r * D + 3 + c] = T[r * D + 3 + c] + dt * T[r * D + 12 + c];
    }
    for (int i = 0; i < 3; i++) {
        P[(15 + i) * D + 15 + i] += cov_gyr_scale[i] * dt * dt;
        P[(12 + i) * D + 12 + i] += cov_acc_scale[i] * dt * dt;
    }
    double Ef[9], R[9];
    so3_exp_dt(s->bias_g, dt, Ef);   // Exp(state_inout.bias_g, dt) (IMU_Processing.hpp:239)
    mul33(s->rot_end, Ef, R);
    std::memcpy(s->rot_end, R, sizeof(R));
    for (int i = 0; i < 3; i++) s->pos_end[i] += s->vel_end[i] * dt;
}

void liinit_imu_init(liinit_imu* imu) {
    std::memset(imu, 0, sizeof(*imu));
    for (int i = 0; i < 3; i++) {
        imu->cov_acc[i] = imu->cov_gyr[i] = 0.1;                 // IMU_Processing.hpp:97-102
        imu->cov_R_LI[i] = 0.00001;
        imu->cov_T_LI[i] = 0.0001;
        imu->cov_bias_gyr[i] = imu->cov_bias_acc[i] = 0.0001;
        imu->cov_acc_scale[i] = imu->cov_gyr_scale[i] = 0.1;     // the node's gyr_cov / acc_cov defaults (laserMapping.cpp:76)
    }
    imu->mean_acc_norm = 9.81;                                   // the node's mean_acc_norm default (:94)
    imu->need_init = 1;
}

void liinit_imu_set_gyr_cov(liinit_imu* imu, const double* v) { std::memcpy(imu->cov_gyr_scale, v, 3 * sizeof(double)); }
void liinit_imu_set_acc_cov(liinit_imu* imu, const double* v) { std::memcpy(imu->cov_acc_scale, v, 3 * sizeof(double)); }
void liinit_imu_set_R_LI_cov(liinit_imu* imu, const double* v) { std::memcpy(imu->cov_R_LI, v, 3 * sizeof(double)); }
void liinit_imu_set_T_LI_cov(liinit_imu* imu, const double* v) { std::memcpy(imu->cov_T_LI, v, 3 * sizeof(double)); }
void liinit_imu_set_gyr_bias_cov(liinit_imu* imu, const double* v) { std::memcpy(imu->cov_bias_gyr, v, 3 * sizeof(double)); }
void liinit_imu_set_acc_bias_cov(liinit_imu* imu, const double* v) { std::memcpy(imu->cov_bias_acc, v, 3 * sizeof(double)); }
void liinit_imu_set_mean_acc_norm(liinit_imu* imu, double m) { imu->mean_acc_norm = m; }

int liinit_imu_switch(liinit_imu* imu, const double* smp, int n) {
    if (!imu || n < 0 || (n > 0 && !smp)) return LIINIT_ERR_INVALID;
    if (n == 0) return LIINIT_OK;
    std::memcpy(imu->last_imu, smp + (size_t)(n - 1) * LIINIT_IMU_SAMPLE_DOUBLES, sizeof(imu->last_imu));   // :448-451
    imu->need_init = 0;
    std::memcpy(imu->cov_acc, imu->cov_acc_scale, sizeof(imu->cov_acc));
    std::memcpy(imu->cov_gyr, imu->cov_gyr_scale, sizeof(imu->cov_gyr));
    return LIINIT_OK;
}

static void put_pose6d(double* o, double t, const double* a, const double* g, const double* v, const double* p, const double* R) {
    o[0] = t;   // set_pose6d (common_lib.h:184-199)
    for (int i = 0; i < 3; i++) {
        o[1 + i] = a[i];
        o[4 + i] = g[i];
        o[7 + i] = v[i];
        o[10 + i] = p[i];
    }
    std::memcpy(o + 13, R, 9 * sizeof(double));
}

int liinit_imu_propagate(liinit_imu* imu, liinit_state* s, const double* smp, int n, double pcl_beg_time, double pcl_end_offset_ms,
                         double* poses, int* npose) {
    if (!imu || !s || !npose || n < 0 || (n > 0 && (!smp || !poses))) return LIINIT_ERR_INVALID;
    *npose = 0;
    if (n == 0) return LIINIT_OK;
    if (imu->need_init) return LIINIT_ERR_INVALID;
    const double G_m_s2 = 9.81;   // common_lib.h:23
    const double last_end = imu->last_lidar_end_time;
    // v_imu = {last_imu_, samples...} (IMU_Processing.hpp:273-274); pair k = (v_imu[k], v_imu[k + 1])
    auto sample = [&](int k) { return k == 0 ? imu->last_imu : smp + (size_t)(k - 1) * LIINIT_IMU_SAMPLE_DOUBLES; };
    int np = 1;
    for (int k = 0; k < n; k++) np += !(sample(k + 1)[0] < last_end);
    if (np > LIINIT_MAX_IMU_POSES) return LIINIT_ERR_CAPACITY;
    const double imu_end_time = sample(n)[0];
    const double pcl_end_time = pcl_beg_time + pcl_end_offset_ms / double(1000);   // :288

    put_pose6d(poses, 0.0, imu->acc_s_last, imu->angvel_last, s->vel_end, s->pos_end, s->rot_end);   // :293-294
    double R[9], vel[3], pos[3], acc_imu[3] = {0, 0, 0}, angvel[3] = {0, 0, 0};   // (never read unset: the table would have one pose)
    std::memcpy(R, s->rot_end, sizeof(R));
    std::memcpy(vel, s->vel_end, sizeof(vel));
    std::memcpy(pos, s->pos_end, sizeof(pos));
    double* P = s->cov;
    double T[D * D];
    int out = 1;
    for (int k = 0; k < n; k++) {
        const double* head = sample(k);
        const double* tail = sample(k + 1);
        if (tail[0] < last_end) continue;   // :307
        double acc[3];
        for (int i = 0; i < 3; i++) {
            angvel[i] = 0.5 * (head[1 + i] + tail[1 + i]);
            acc[i] = 0.5 * (head[4 + i] + tail[4 + i]);
            angvel[i] -= s->bias_g[i];                                   // :322
            acc[i] = acc[i] / imu->mean_acc_norm * G_m_s2 - s->bias_a[i];   // :323
        }
        const double dt = (head[0] < last_end) ? tail[0] - last_end : tail[0] - head[0];   // :325-328
        double Ef[9], Eb[9];
        so3_exp_dt(angvel, dt, Ef);
        so3_exp_dt(angvel, -dt, Eb);
        // F (:335-343) is the identity except in rows 0:3 (Exp(-dt) at 0, -dt I at 15), 3:6 (dt I at 12) and 12:15
        // (A = -R [acc]x dt at 0, -R dt at 18, dt I at 21). F P F^T is formed as T = F P, then T F^T; both sum in column order.
        const double K[9] = {0, -acc[2], acc[1], acc[2], 0, -acc[0], -acc[1], acc[0], 0};
        double nR[9], A[9], B[9];
        for (int i = 0; i < 9; i++) nR[i] = -R[i];
        mul33(nR, K, A);
        for (int i = 0; i < 9; i++) {
            A[i] *= dt;
            B[i] = nR[i] * dt;
        }
        std::memcpy(T, P, sizeof(T));
        for (int c = 0; c < D; c++)
            for (int i = 0; i < 3; i++) {
                T[i * D + c] = Eb[3 * i] * P[c] + Eb[3 * i + 1] * P[D + c] + Eb[3 * i + 2] * P[2 * D + c] + (-dt) * P[(15 + i) * D + c];
                T[(3 + i) * D + c] = P[(3 + i) * D + c] + dt * P[(12 + i) * D + c];
                T[(12 + i) * D + c] = A[3 * i] * P[c] + A[3 * i + 1] * P[D + c] + A[3 * i + 2] * P[2 * D + c] + P[(12 + i) * D + c] +
                                      B[3 * i] * P[18 * D + c] + B[3 * i + 1] * P[19 * D + c] + B[3 * i + 2] * P[20 * D + c] +
                                      dt * P[(21 + i) * D + c];
            }
        std::memcpy(P, T, sizeof(T));
        for (int r = 0; r < D; r++) {
            const double* t = T + r * D;
            for (int i = 0; i < 3; i++) {
                P[r * D + i] = t[0] * Eb[3 * i] + t[1] * Eb[3 * i + 1] + t[2] * Eb[3 * i + 2] + t[15 + i] * (-dt);
                P[r * D + 3 + i] = t[3 + i] + t[12 + i] * dt;
                P[r * D + 12 + i] = t[0] * A[3 * i] + t[1] * A[3 * i + 1] + t[2] * A[3 * i + 2] + t[12 + i] + t[18] * B[3 * i] +
                                    t[19] * B[3 * i + 1] + t[20] * B[3 * i + 2] + t[21 + i] * dt;
            }
        }
        // Q (:345-350); the acceleration block is R diag(cov_acc) R^T dt^2
        for (int i = 0; i < 3; i++) {
            P[i * D + i] += imu->cov_gyr[i] * dt * dt;
            P[(6 + i) * D + 6 + i] += imu->cov_R_LI[i] * dt * dt;
            P[(9 + i) * D + 9 + i] += imu->cov_T_LI[i] * dt * dt;
            P[(15 + i) * D + 15 + i] += imu->cov_bias_gyr[i] * dt * dt;
            P[(18 + i) * D + 18 + i] += imu->cov_bias_acc[i] * dt * dt;
            for (int j = 0; j < 3; j++) {
                double q = R[3 * i] * imu->cov_acc[0] * R[3 * j] + R[3 * i + 1] * imu->cov_acc[1] * R[3 * j + 1] +
                           R[3 * i + 2] * imu->cov_acc[2] * R[3 * j + 2];
                P[(12 + i) * D + 12 + j] += q * dt * dt;
            }
        }
        double Rn[9];   // :355-364
        mul33(R, Ef, Rn);
        std::memcpy(R, Rn, sizeof(R));
        for (int i = 0; i < 3; i++) acc_imu[i] = R[3 * i] * acc[0] + R[3 * i + 1] * acc[1] + R[3 * i + 2] * acc[2] + s->gravity[i];
        for (int i = 0; i < 3; i++) {
            pos[i] = pos[i] + vel[i] * dt + 0.5 * acc_imu[i] * dt * dt;
            vel[i] = vel[i] + acc_imu[i] * dt;
        }
        std::memcpy(imu->angvel_last, angvel, sizeof(angvel));   // :367-370
        std::memcpy(imu->acc_s_last, acc_imu, sizeof(acc_imu));
        put_pose6d(poses + (size_t)out * LIINIT_POSE6D_DOUBLES, tail[0] - pcl_beg_time, acc_imu, angvel, vel, pos, R);
        out++;
    }
    // extrapolation to the scan end, forwards (note = 1) or backwards (note = -1) from the last sample (:374-378)
    const double note = pcl_end_time > imu_end_time ? 1.0 : -1.0;
    const double dt = note * (pcl_end_time - imu_end_time);
    const double w[3] = {note * angvel[0], note * angvel[1], note * angvel[2]};
    double E[9];
    so3_exp_dt(w, dt, E);
    mul33(R, E, s->rot_end);
    for (int i = 0; i < 3; i++) {
        s->vel_end[i] = vel[i] + note * acc_imu[i] * dt;
        s->pos_end[i] = pos[i] + note * vel[i] * dt + note * 0.5 * acc_imu[i] * dt * dt;
    }
    std::memcpy(imu->last_imu, sample(n), sizeof(imu->last_imu));   // :381-382
    imu->last_lidar_end_time = pcl_end_time;
    *npose = out;
    return LIINIT_OK;
}

int liinit_replay_run(liinit_ctx* h, const liinit_replay_job* job, liinit_state* states, int* frames, int cap, int* n_updates) {
    if (!h || !job || !n_updates || cap < 0 || (cap > 0 && (!states || !frames)) || job->n_buf < 0 || job->n_samples < 0 || job->n_events < 0 ||
        (job->n_buf > 0 && !job->buf_rows) || (job->n_samples > 0 && !job->samples) || (job->n_events > 0 && !job->events) || job->max_iteration < 1)
        return LIINIT_ERR_INVALID;
    *n_updates = 0;
    constexpr int W = LIINIT_IMU_SAMPLE_DOUBLES;
    using Row = std::array<double, W>;
    liinit_state s = job->state;
    liinit_imu imu = job->imu;
    std::deque<Row> rows;   // ImuBuffer.rows
    for (int i = 0; i < job->n_buf; i++) {
        Row r;
        std::memcpy(r.data(), job->buf_rows + (size_t)i * W, sizeof(Row));
        rows.push_back(r);
    }
    double last_stamp = job->last_stamp;
    int frame_num = job->frame_num, switch_scan = job->switch_scan, next_sample = 0;
    std::deque<int> pending;
    std::vector<double> group, poses;
    for (int e = 0; e < job->n_events; e++) {
        const int ev = job->events[e];
        if (ev >= 0) {
            pending.push_back(ev);
        } else if (ev == LIINIT_REPLAY_IMU && next_sample < job->n_samples) {
            // ImuBuffer.push: imu_cbk's time compensation and its loop-back clear (laserMapping.cpp:412-423)
            const double* x = job->samples + (size_t)next_sample++ * W;
            Row r;
            std::memcpy(r.data(), x, sizeof(Row));
            r[0] = x[0] - job->timediff - job->time_lag;
            if (r[0] < last_stamp) rows.clear();
            last_stamp = r[0];
            rows.push_back(r);
        } else {
            return LIINIT_ERR_INVALID;
        }
        while (!pending.empty()) {
            const int j = pending.front();
            double t_beg;
            float end_ms;
            int rc = liinit_replay_frame(h, j, &t_beg, &end_ms, nullptr);
            if (rc != LIINIT_OK) return rc;
            const double t_end = t_beg + (double)end_ms / 1000.0;   // lidar_end_time
            if (rows.empty() || !(last_stamp >= t_end)) break;     // sync_packages waits for an IMU stamp >= lidar_end_time
            pending.pop_front();
            // ImuBuffer.pop: the measure group, the buffered samples with stamp <= lidar_end_time (:466-474)
            group.clear();
            double imu_time = rows.empty() ? 0.0 : rows.front()[0];
            while (!rows.empty() && imu_time < t_end) {
                imu_time = rows.front()[0];
                if (imu_time > t_end) break;
                group.insert(group.end(), rows.front().begin(), rows.front().end());
                rows.pop_front();
            }
            const int n = (int)(group.size() / W);
            // process_raw in LIO mode
            if (n && !imu.need_init) {
                poses.resize((size_t)(n + 1) * LIINIT_POSE6D_DOUBLES);
                int np = 0;
                rc = liinit_imu_propagate(&imu, &s, group.data(), n, t_beg, (double)end_ms, poses.data(), &np);
                if (rc != LIINIT_OK) return rc;
                rc = liinit_replay_stage(h, j);
                if (rc != LIINIT_OK) return rc;
                if (np >= 2) {
                    rc = liinit_raw_undistort_imu(h, poses.data(), np, s.rot_end, s.pos_end, s.offset_R_L_I, s.offset_T_L_I);
                    if (rc != LIINIT_OK) return rc;
                }
            } else if (n) {
                rc = liinit_imu_switch(&imu, group.data(), n);   // the switch scan: the previous cloud is matched again
                if (rc != LIINIT_OK) return rc;
                switch_scan = frame_num;
            }
            int n_down = 0, n_add = 0, n_nd = 0;
            rc = liinit_raw_downsample(h, (float)job->filter_size_surf, &n_down);
            if (rc != LIINIT_OK) return rc;
            rc = scan_update(h, &s, job->max_iteration, 1, nullptr, job->frozen != 0);
            if (rc != LIINIT_OK) return rc;
            rc = liinit_map_incremental(h, s.rot_end, s.pos_end, s.offset_R_L_I, s.offset_T_L_I, job->filter_size_map, 1, &n_add, &n_nd);
            if (rc != LIINIT_OK) return rc;
            frame_num++;
            if (*n_updates >= cap) return LIINIT_ERR_CAPACITY;
            states[*n_updates] = s;
            frames[*n_updates] = j;
            ++*n_updates;
            if (switch_scan != frame_num - 1) {
                int appended = 0;
                rc = liinit_assess_append(h, s.rot_end, s.pos_end, s.offset_R_L_I, s.offset_T_L_I, &appended);
                if (rc != LIINIT_OK) return rc;
            }
        }
    }
    return LIINIT_OK;
}

int liinit_fov_segment(const double* pos, double cube_len, double det_range, float* box, int* initialized, float* out) {
    const double MOV_THRESHOLD = 1.5;   // laserMapping.cpp:58
    if (!*initialized) {                 // :266-272
        for (int i = 0; i < 3; i++) {
            box[i] = (float)(pos[i] - cube_len / 2.0);
            box[3 + i] = (float)(pos[i] + cube_len / 2.0);
        }
        *initialized = 1;
        return 0;
    }
    float dist[3][2];
    bool need_move = false;
    for (int i = 0; i < 3; i++) {        // :274-281
        dist[i][0] = (float)std::fabs(pos[i] - (double)box[i]);
        dist[i][1] = (float)std::fabs(pos[i] - (double)box[3 + i]);
        if (dist[i][0] <= MOV_THRESHOLD * det_range || dist[i][1] <= MOV_THRESHOLD * det_range) need_move = true;
    }
    if (!need_move) return 0;
    float nb[6];
    std::memcpy(nb, box, sizeof(nb));
    const double a = (cube_len - 2.0 * MOV_THRESHOLD * det_range) * 0.5 * 0.9, b = det_range * (MOV_THRESHOLD - 1);
    const float mov_dist = (float)(a > b ? a : b);   // :285-286
    int n = 0;
    for (int i = 0; i < 3; i++) {        // :287-301
        float tmp[6];
        std::memcpy(tmp, box, sizeof(tmp));
        if (dist[i][0] <= MOV_THRESHOLD * det_range) {
            nb[3 + i] -= mov_dist;
            nb[i] -= mov_dist;
            tmp[i] = box[3 + i] - mov_dist;
            std::memcpy(out + 6 * n++, tmp, sizeof(tmp));
        } else if (dist[i][1] <= MOV_THRESHOLD * det_range) {
            nb[3 + i] += mov_dist;
            nb[i] += mov_dist;
            tmp[3 + i] = box[i] + mov_dist;
            std::memcpy(out + 6 * n++, tmp, sizeof(tmp));
        }
    }
    std::memcpy(box, nb, sizeof(nb));
    return n;
}

}  // extern "C"
