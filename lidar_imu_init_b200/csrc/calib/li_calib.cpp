// li_calib.cpp -- LI-Init batch initialisation on the host (SURVEY.md 8f row N4; C-ABI in include/liinit_calib.h).
//
// Restates the data flow of the reference's LI_Init class (include/LI_init/LI_init.cpp) stage by stage -- the sample
// bookkeeping (which elements are dropped, shifted, interpolated) decides the result as much as the solvers do, so it
// is followed literally, including its quirks:
//   * "all but the last element" loops (:28,:32,:44,:48,:209) and the 10 / 20 element cuts (:197-204, :224-228);
//   * the filter extension mirrors 60 samples without repeating the edge sample, starts the recursion at index 7 with
//     unfiltered history, and leaves time stamps / rotations untouched (:260-304);
//   * the running-mean forms (x += (v - x) / k) of :97-99, :164-167, :497-499.
// Not restated: Ceres. The three non-linear least-squares problems (:317-343, :345-395, :403-474) are solved by
// Levenberg-Marquardt on SO(3) x R^n run to convergence (the reference stops Ceres at its default tolerances, so its
// printed values sit within those tolerances of the optimum computed here). The box constraint on the accelerometer
// bias (:448-451) is kept by an active-set projection.
// One deviation: the 5-tap mean filter of :92-99 reads one element past the end of its source copy for the last
// filtered sample; here that tap reads the last sample of the full buffer.
#include "liinit_calib.h"

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <deque>
#include <vector>

namespace {

constexpr double kG = 9.81;   // G_m_s2, include/common_lib.h:23

struct V3 {
    double x = 0, y = 0, z = 0;
    V3() {}
    V3(double a, double b, double c) : x(a), y(b), z(c) {}
    V3 operator+(const V3& o) const { return V3(x + o.x, y + o.y, z + o.z); }
    V3 operator-(const V3& o) const { return V3(x - o.x, y - o.y, z - o.z); }
    V3 operator*(double s) const { return V3(x * s, y * s, z * s); }
    V3 operator/(double s) const { return V3(x / s, y / s, z / s); }
    double norm() const { return std::sqrt(x * x + y * y + z * z); }
    double operator[](int i) const { return i == 0 ? x : (i == 1 ? y : z); }
};

struct M3 {
    double m[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    double& operator()(int r, int c) { return m[3 * r + c]; }
    double operator()(int r, int c) const { return m[3 * r + c]; }
    V3 operator*(const V3& v) const {
        return V3(m[0] * v.x + m[1] * v.y + m[2] * v.z, m[3] * v.x + m[4] * v.y + m[5] * v.z, m[6] * v.x + m[7] * v.y + m[8] * v.z);
    }
    M3 operator*(const M3& o) const {
        M3 r;
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) r(i, j) = m[3 * i] * o(0, j) + m[3 * i + 1] * o(1, j) + m[3 * i + 2] * o(2, j);
        return r;
    }
    M3 t() const {
        M3 r;
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) r(i, j) = m[3 * j + i];
        return r;
    }
};
M3 skew(const V3& v) {
    M3 s;
    s(0, 0) = 0; s(0, 1) = -v.z; s(0, 2) = v.y;
    s(1, 0) = v.z; s(1, 1) = 0; s(1, 2) = -v.x;
    s(2, 0) = -v.y; s(2, 1) = v.x; s(2, 2) = 0;
    return s;
}
M3 madd(const M3& a, const M3& b) {
    M3 r;
    for (int i = 0; i < 9; i++) r.m[i] = a.m[i] + b.m[i];
    return r;
}
// Rodrigues
M3 so3_exp(const V3& w) {
    double th = w.norm();
    M3 R;
    if (th < 1e-12) return madd(R, skew(w));
    V3 a = w / th;
    M3 K = skew(a), K2 = K * K;
    double s = std::sin(th), c = 1 - std::cos(th);
    for (int i = 0; i < 9; i++) R.m[i] += s * K.m[i] + c * K2.m[i];
    return R;
}
// nearest rotation by one quaternion round trip (keeps the LM iterate on the manifold)
M3 renorm(const M3& R) {
    double q[4];
    double tr = R(0, 0) + R(1, 1) + R(2, 2);
    if (tr > 0) {
        double s = std::sqrt(tr + 1.0) * 2;
        q[0] = 0.25 * s; q[1] = (R(2, 1) - R(1, 2)) / s; q[2] = (R(0, 2) - R(2, 0)) / s; q[3] = (R(1, 0) - R(0, 1)) / s;
    } else if (R(0, 0) > R(1, 1) && R(0, 0) > R(2, 2)) {
        double s = std::sqrt(1.0 + R(0, 0) - R(1, 1) - R(2, 2)) * 2;
        q[0] = (R(2, 1) - R(1, 2)) / s; q[1] = 0.25 * s; q[2] = (R(0, 1) + R(1, 0)) / s; q[3] = (R(0, 2) + R(2, 0)) / s;
    } else if (R(1, 1) > R(2, 2)) {
        double s = std::sqrt(1.0 + R(1, 1) - R(0, 0) - R(2, 2)) * 2;
        q[0] = (R(0, 2) - R(2, 0)) / s; q[1] = (R(0, 1) + R(1, 0)) / s; q[2] = 0.25 * s; q[3] = (R(1, 2) + R(2, 1)) / s;
    } else {
        double s = std::sqrt(1.0 + R(2, 2) - R(0, 0) - R(1, 1)) * 2;
        q[0] = (R(1, 0) - R(0, 1)) / s; q[1] = (R(0, 2) + R(2, 0)) / s; q[2] = (R(1, 2) + R(2, 1)) / s; q[3] = 0.25 * s;
    }
    double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    double w = q[0] / n, x = q[1] / n, y = q[2] / n, z = q[3] / n;
    M3 o;
    o(0, 0) = 1 - 2 * (y * y + z * z); o(0, 1) = 2 * (x * y - z * w); o(0, 2) = 2 * (x * z + y * w);
    o(1, 0) = 2 * (x * y + z * w); o(1, 1) = 1 - 2 * (x * x + z * z); o(1, 2) = 2 * (y * z - x * w);
    o(2, 0) = 2 * (x * z - y * w); o(2, 1) = 2 * (y * z + x * w); o(2, 2) = 1 - 2 * (x * x + y * y);
    return o;
}
// RotMtoEuler, include/so3_math.h:110-131
V3 rot_to_euler(const M3& r) {
    double sy = std::sqrt(r(0, 0) * r(0, 0) + r(1, 0) * r(1, 0));
    if (sy >= 1e-6) return V3(std::atan2(r(2, 1), r(2, 2)), std::atan2(-r(2, 0), sy), std::atan2(r(1, 0), r(0, 0)));
    return V3(std::atan2(-r(1, 2), r(1, 1)), std::atan2(-r(2, 0), sy), 0);
}

// CalibState, LI_init.h:30-89. The arithmetic operators of the reference touch only the four vectors below;
// rot / t travel with copies only.
struct Sample {
    M3 rot;
    V3 w, v, wa, va;   // ang_vel, linear_vel, ang_acc, linear_acc
    double t = 0;
};
typedef std::deque<Sample> Seq;

// ---- dense symmetric solve (n <= 9): Cholesky, tiny pivots lifted (the yaw of R_GL0 is a gauge direction) ----
bool chol_solve(int n, const double* A, const double* b, double* x) {
    double L[81];
    for (int i = 0; i < n; i++) {
        for (int j = 0; j <= i; j++) {
            double s = A[i * n + j];
            for (int k = 0; k < j; k++) s -= L[i * n + k] * L[j * n + k];
            if (i == j) {
                if (!(s > 0)) return false;
                L[i * n + i] = std::sqrt(s);
            } else {
                L[i * n + j] = s / L[j * n + j];
            }
        }
    }
    double y[9];
    for (int i = 0; i < n; i++) {
        double s = b[i];
        for (int k = 0; k < i; k++) s -= L[i * n + k] * y[k];
        y[i] = s / L[i * n + i];
    }
    for (int i = n - 1; i >= 0; i--) {
        double s = y[i];
        for (int k = i + 1; k < n; k++) s -= L[k * n + i] * x[k];
        x[i] = s / L[i * n + i];
    }
    return true;
}

// ---- Levenberg-Marquardt over x = (R in SO(3), p in R^np), local step d = (dtheta, dp): R <- Exp(dtheta) R ------
struct Problem {
    int np = 0;                                   // Euclidean parameters after the rotation
    double lo[6], hi[6];                          // box on p (+-inf when free)
    // cost = 0.5 * sum r^2; fills JtJ [(3+np)^2] and Jtr [(3+np)] when asked
    virtual double eval(const M3& R, const double* p, double* JtJ, double* Jtr) const = 0;
    virtual ~Problem() {}
};

int lm_solve(const Problem& P, M3& R, double* p, double* final_cost) {
    const int n = 3 + P.np;
    double JtJ[81], g[9];
    double cost = P.eval(R, p, JtJ, g);
    double lambda = 1e-4;
    int it = 0;
    for (; it < 500; it++) {
        // active set: a bounded parameter sitting on its bound with the descent direction pointing outwards is frozen
        bool frozen[9] = {false};
        for (int k = 0; k < P.np; k++) {
            if (p[k] <= P.lo[k] && g[3 + k] > 0) frozen[3 + k] = true;
            if (p[k] >= P.hi[k] && g[3 + k] < 0) frozen[3 + k] = true;
        }
        int idx[9], nf = 0;
        for (int k = 0; k < n; k++)
            if (!frozen[k]) idx[nf++] = k;
        double gn = 0;
        for (int a = 0; a < nf; a++) gn = std::max(gn, std::fabs(g[idx[a]]));
        if (gn < 1e-13 * (1.0 + cost)) break;
        bool accepted = false;
        double step_norm = 0;
        for (int tries = 0; tries < 60 && !accepted; tries++) {
            double A[81], b[9], d[9];
            for (int a = 0; a < nf; a++) {
                for (int c = 0; c < nf; c++) A[a * nf + c] = JtJ[idx[a] * n + idx[c]];
                double dd = JtJ[idx[a] * n + idx[a]];
                A[a * nf + a] += lambda * (dd > 1e-12 ? dd : 1e-12);
                b[a] = -g[idx[a]];
            }
            if (!chol_solve(nf, A, b, d)) {
                lambda *= 10;
                continue;
            }
            double full[9] = {0};
            for (int a = 0; a < nf; a++) full[idx[a]] = d[a];
            M3 Rn = renorm(so3_exp(V3(full[0], full[1], full[2])) * R);
            double pn[6];
            for (int k = 0; k < P.np; k++) pn[k] = std::min(P.hi[k], std::max(P.lo[k], p[k] + full[3 + k]));
            double cn = P.eval(Rn, pn, nullptr, nullptr);
            if (cn <= cost) {
                step_norm = 0;
                for (int k = 0; k < 3; k++) step_norm = std::max(step_norm, std::fabs(full[k]));
                for (int k = 0; k < P.np; k++) step_norm = std::max(step_norm, std::fabs(pn[k] - p[k]));
                R = Rn;
                for (int k = 0; k < P.np; k++) p[k] = pn[k];
                double dec = cost - cn;
                cost = cn;
                lambda = std::max(lambda * 0.2, 1e-12);
                accepted = true;
                if (dec <= 1e-16 * (1.0 + cost)) step_norm = 0;   // no measurable progress left
            } else {
                lambda *= 4;
            }
        }
        if (!accepted) break;
        cost = P.eval(R, p, JtJ, g);
        if (step_norm < 1e-14) break;
    }
    if (final_cost) *final_cost = cost;
    return it;
}

// ---- the reference's solver schedule ---------------------------------------------------------------------------
// The reference calls ceres::Solve with default options (LI_init.cpp:336-339, :383-385, :453-455): trust-region
// Levenberg-Marquardt, Jacobi scaling fixed at the first iterate, initial radius 1e4, LM diagonal clamped to
// [1e-6, 1e32], radius / max(1/3, 1 - (2 rho - 1)^3) after a good step (rho > 1e-3), halved with a doubling factor
// after a bad one, at most 50 iterations, and -- what fixes the printed digits -- termination as soon as a candidate
// changes the cost by less than 1e-6 * cost, WITHOUT taking that candidate. Its quaternion block moves by
// q <- [cos|d|, sin|d| d/|d|] (x) q, i.e. a left rotation by 2d. Following that schedule (not Ceres' code) lands on
// the same iterate as the reference instead of the exact optimum a few 1e-5 away.
struct Quat {
    double w = 1, x = 0, y = 0, z = 0;
};
M3 quat_to_rot(const Quat& q) {
    const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
    const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
    const double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x, tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
    M3 R;
    R(0, 0) = 1 - (tyy + tzz); R(0, 1) = txy - twz; R(0, 2) = txz + twy;
    R(1, 0) = txy + twz; R(1, 1) = 1 - (txx + tzz); R(1, 2) = tyz - twx;
    R(2, 0) = txz - twy; R(2, 1) = tyz + twx; R(2, 2) = 1 - (txx + tyy);
    return R;
}
Quat quat_plus(const Quat& q, const double d[3]) {
    const double nd = std::sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    if (!(nd > 0)) return q;
    const double sc = std::sin(nd) / nd;
    const double a = std::cos(nd), b = sc * d[0], c = sc * d[1], e = sc * d[2];   // q_delta
    Quat o;                                                                        // q_delta (x) q
    o.w = a * q.w - b * q.x - c * q.y - e * q.z;
    o.x = a * q.x + b * q.w + c * q.z - e * q.y;
    o.y = a * q.y - b * q.z + c * q.w + e * q.x;
    o.z = a * q.z + b * q.y - c * q.x + e * q.w;
    return o;
}

int tr_solve_reference_schedule(const Problem& P, Quat& q, double* p, double* final_cost) {
    const int n = 3 + P.np;
    double A[81], g[9], scale[9];
    auto linearize = [&](const Quat& qq, const double* pp) {
        double c = P.eval(quat_to_rot(qq), pp, A, g);
        for (int a = 0; a < n; a++) {   // rotation columns are per unit of d, the rotation vector is 2d
            const double sa = a < 3 ? 2.0 : 1.0;
            g[a] *= sa;
            for (int b = 0; b < n; b++) A[a * n + b] *= sa * (b < 3 ? 2.0 : 1.0);
        }
        return c;
    };
    double cost = linearize(q, p);
    for (int a = 0; a < n; a++) scale[a] = 1.0 / (1.0 + std::sqrt(A[a * n + a]));
    double radius = 1e4, decrease = 2.0;
    int it = 0;
    for (it = 1; it <= 50; it++) {
        double As[81], gs[9], M[81], rhs[9], s[9];
        for (int a = 0; a < n; a++) {
            gs[a] = g[a] * scale[a];
            for (int b = 0; b < n; b++) As[a * n + b] = A[a * n + b] * scale[a] * scale[b];
        }
        std::memcpy(M, As, sizeof(double) * n * n);
        for (int a = 0; a < n; a++) {
            M[a * n + a] += std::min(std::max(As[a * n + a], 1e-6), 1e32) / radius;
            rhs[a] = -gs[a];
        }
        bool ok = chol_solve(n, M, rhs, s);
        double model = 0;
        if (ok) {
            for (int a = 0; a < n; a++) {
                double As_s = 0;
                for (int b = 0; b < n; b++) As_s += As[a * n + b] * s[b];
                model -= s[a] * (gs[a] + 0.5 * As_s);
            }
        }
        if (!ok || !(model > 0)) {   // invalid step: shrink and retry
            radius /= decrease;
            decrease *= 2;
            continue;
        }
        double d[9];
        for (int a = 0; a < n; a++) d[a] = s[a] * scale[a];
        Quat qc = quat_plus(q, d);
        double pc[6];
        for (int k = 0; k < P.np; k++) pc[k] = std::min(P.hi[k], std::max(P.lo[k], p[k] + d[3 + k]));
        const double cc = P.eval(quat_to_rot(qc), pc, nullptr, nullptr);
        // parameter tolerance on the ambient step
        double sn = (qc.w - q.w) * (qc.w - q.w) + (qc.x - q.x) * (qc.x - q.x) + (qc.y - q.y) * (qc.y - q.y) + (qc.z - q.z) * (qc.z - q.z);
        double xn = q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z;
        for (int k = 0; k < P.np; k++) { sn += (pc[k] - p[k]) * (pc[k] - p[k]); xn += p[k] * p[k]; }
        if (std::sqrt(sn) <= 1e-8 * (std::sqrt(xn) + 1e-8)) break;
        if (std::fabs(cost - cc) <= 1e-6 * cost) break;           // function tolerance: candidate not taken
        const double rho = (cost - cc) / model;
        if (rho > 1e-3) {
            q = qc;
            for (int k = 0; k < P.np; k++) p[k] = pc[k];
            cost = linearize(q, p);
            radius = std::min(1e16, radius / std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * rho - 1.0, 3)));
            decrease = 2.0;
            double gmax = 0;
            for (int a = 0; a < n; a++) gmax = std::max(gmax, std::fabs(g[a]));
            if (gmax <= 1e-10) break;
        } else {
            radius /= decrease;
            decrease *= 2;
        }
    }
    if (final_cost) *final_cost = cost;
    return it;
}

void add_block(double* JtJ, double* Jtr, int n, const double (*J)[9], const double* r) {   // J: 3 x n rows
    for (int a = 0; a < n; a++) {
        double ga = J[0][a] * r[0] + J[1][a] * r[1] + J[2][a] * r[2];
        Jtr[a] += ga;
        for (int c = a; c < n; c++) JtJ[a * n + c] += J[0][a] * J[0][c] + J[1][a] * J[1][c] + J[2][a] * J[2][c];
    }
}
void symmetrize(double* JtJ, int n) {
    for (int a = 0; a < n; a++)
        for (int c = 0; c < a; c++) JtJ[a * n + c] = JtJ[c * n + a];
}

// Angular_Vel_Cost_only_Rot (LI_init.h:91-117): r = R w_L - w_I
struct RotOnly : Problem {
    const Seq *I, *L;
    double eval(const M3& R, const double*, double* JtJ, double* Jtr) const override {
        const int n = 3;
        if (JtJ) { std::fill(JtJ, JtJ + n * n, 0.0); std::fill(Jtr, Jtr + n, 0.0); }
        double c = 0;
        for (size_t i = 0; i < I->size(); i++) {
            V3 a = R * (*L)[i].w;
            V3 r = a - (*I)[i].w;
            c += r.x * r.x + r.y * r.y + r.z * r.z;
            if (JtJ) {
                M3 S = skew(a);   // d(Exp(d) a)/dd = -[a]x
                double J[3][9], rr[3] = {r.x, r.y, r.z};
                for (int k = 0; k < 3; k++)
                    for (int q = 0; q < 3; q++) J[k][q] = -S(k, q);
                add_block(JtJ, Jtr, n, J, rr);
            }
        }
        if (JtJ) symmetrize(JtJ, n);
        return 0.5 * c;
    }
};

// Angular_Vel_Cost (LI_init.h:119-160): r = R w_L - w_I - (dT_i + td) a_I + b_g ; p = [b_g(3), td]
struct RotBias : Problem {
    const Seq *I, *L;
    double eval(const M3& R, const double* p, double* JtJ, double* Jtr) const override {
        const int n = 7;
        if (JtJ) { std::fill(JtJ, JtJ + n * n, 0.0); std::fill(Jtr, Jtr + n, 0.0); }
        double c = 0;
        V3 bg(p[0], p[1], p[2]);
        for (size_t i = 0; i < I->size(); i++) {
            double dT = (*L)[i].t - (*I)[i].t;
            V3 a = R * (*L)[i].w;
            V3 r = a - (*I)[i].w - (*I)[i].wa * (dT + p[3]) + bg;
            c += r.x * r.x + r.y * r.y + r.z * r.z;
            if (JtJ) {
                M3 S = skew(a);
                double J[3][9], rr[3] = {r.x, r.y, r.z};
                for (int k = 0; k < 3; k++) {
                    for (int q = 0; q < 3; q++) { J[k][q] = -S(k, q); J[k][3 + q] = (k == q) ? 1.0 : 0.0; }
                    J[k][6] = -(*I)[i].wa[k];
                }
                add_block(JtJ, Jtr, n, J, rr);
            }
        }
        if (JtJ) symmetrize(JtJ, n);
        return 0.5 * c;
    }
};

// Linear_acc_Cost (LI_init.h:162-205): r = R_i R_LI^T a_I - R_i b_a + R_G g - a_L - R_i ([w]x^2 + [wa]x) T ; p = [b_a(3), T(3)]
struct TransAcc : Problem {
    const Seq *I, *L;
    M3 R_LI;
    double eval(const M3& RG, const double* p, double* JtJ, double* Jtr) const override {
        const int n = 9;
        if (JtJ) { std::fill(JtJ, JtJ + n * n, 0.0); std::fill(Jtr, Jtr + n, 0.0); }
        double c = 0;
        V3 ba(p[0], p[1], p[2]), T(p[3], p[4], p[5]);
        V3 gv = RG * V3(0, 0, -kG);
        M3 RLIt = R_LI.t();
        M3 Sg = skew(gv);
        for (size_t i = 0; i < I->size(); i++) {
            const Sample& l = (*L)[i];
            M3 Wx = skew(l.w);
            M3 Mi = madd(Wx * Wx, skew(l.wa));
            M3 RM = l.rot * Mi;
            V3 r = l.rot * (RLIt * (*I)[i].va) - l.rot * ba + gv - l.va - RM * T;
            c += r.x * r.x + r.y * r.y + r.z * r.z;
            if (JtJ) {
                double J[3][9], rr[3] = {r.x, r.y, r.z};
                for (int k = 0; k < 3; k++)
                    for (int q = 0; q < 3; q++) { J[k][q] = -Sg(k, q); J[k][3 + q] = -l.rot(k, q); J[k][6 + q] = -RM(k, q); }
                add_block(JtJ, Jtr, n, J, rr);
            }
        }
        if (JtJ) symmetrize(JtJ, n);
        return 0.5 * c;
    }
};

// symmetric 3x3 eigen decomposition (cyclic Jacobi); columns of V are the eigenvectors
void eig_sym3(const double A[9], double w[3], double V[9]) {
    double a[9];
    std::memcpy(a, A, sizeof a);
    for (int i = 0; i < 9; i++) V[i] = (i % 4 == 0) ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 60; sweep++) {
        double off = std::fabs(a[1]) + std::fabs(a[2]) + std::fabs(a[5]);
        if (off < 1e-300) break;
        for (int p = 0; p < 2; p++)
            for (int q = p + 1; q < 3; q++) {
                double apq = a[3 * p + q];
                if (std::fabs(apq) < 1e-300) continue;
                double th = (a[3 * q + q] - a[3 * p + p]) / (2 * apq);
                double t = (th >= 0 ? 1.0 : -1.0) / (std::fabs(th) + std::sqrt(th * th + 1));
                double c = 1 / std::sqrt(t * t + 1), s = t * c;
                for (int k = 0; k < 3; k++) {
                    double akp = a[3 * k + p], akq = a[3 * k + q];
                    a[3 * k + p] = c * akp - s * akq;
                    a[3 * k + q] = s * akp + c * akq;
                }
                for (int k = 0; k < 3; k++) {
                    double apk = a[3 * p + k], aqk = a[3 * q + k];
                    a[3 * p + k] = c * apk - s * aqk;
                    a[3 * q + k] = s * apk + c * aqk;
                }
                for (int k = 0; k < 3; k++) {
                    double vkp = V[3 * k + p], vkq = V[3 * k + q];
                    V[3 * k + p] = c * vkp - s * vkq;
                    V[3 * k + q] = s * vkp + c * vkq;
                }
            }
    }
    w[0] = a[0]; w[1] = a[4]; w[2] = a[8];
}

}  // namespace

struct li_calib {
    Seq imu, lidar, imu_all;            // IMU_state_group, Lidar_state_group, IMU_state_group_ALL (LI_init.h:322-324)
    double data_accum_length = 300;     // LI_init.cpp:17
    double hess_rot[9] = {0};           // Jacobian_rot^T Jacobian_rot, accumulated (laserMapping.cpp:1193-1195)
    M3 R_GL0, R_LI;
    V3 grav_L0, T_LI, bg, ba;
    double lag1 = 0, lag2 = 0, total_lag = 0;
    int lag_frames = 0;
    int solver = 0;   // 0: the reference's ceres-default schedule, 1: Levenberg-Marquardt to convergence
    std::vector<double> log_rows[6];   // li_calib_log_rows: which -> table
};

namespace {

// LI_init.cpp:82-125
void downsample_interpolate(li_calib* c, double move_start_time) {
    Seq& A = c->imu_all;
    while (!A.empty() && A.front().t < move_start_time - 3.0) A.pop_front();
    while (!c->lidar.empty() && c->lidar.front().t < move_start_time - 3.0) c->lidar.pop_front();
    const int n = (int)A.size();
    std::vector<V3> acc0(n);
    for (int i = 0; i < n; i++) acc0[i] = A[i].va;
    const int h = 2;
    for (int i = h; i < n - h; i++) {
        V3 m;
        for (int k = -h; k <= h; k++) m = m + (acc0[i + k] - m) / (double)(k + h + 1);
        A[i].va = m;
    }
    for (size_t i = 0; i < c->lidar.size(); i++) {
        const double tl = c->lidar[i].t;
        for (int j = 1; j < n; j++) {
            if (A[j - 1].t <= tl && A[j].t > tl) {
                double s = (A[j].t - tl) / (A[j].t - A[j - 1].t);
                Sample x;
                x.w = A[j - 1].w * s + A[j].w * (1 - s);
                x.va = A[j - 1].va * s + A[j].va * (1 - s);
                x.t = tl;
                c->imu.push_back(x);
                break;
            }
        }
    }
}

void align_fronts_and_sizes(Seq& I, Seq& L) {   // LI_init.cpp:212-221 == :229-238
    while (!L.empty() && !I.empty() && L.front().t < I.front().t) L.pop_front();
    while (I.size() > 1 && !L.empty() && L.front().t > I[1].t) I.pop_front();
    while (I.size() > L.size()) I.pop_back();
    while (I.size() < L.size()) L.pop_back();
}

// LI_init.cpp:195-221
void time_compensate(li_calib* c, double lag, bool discard) {
    if (discard)
        for (int i = 0; i < 10 && !c->lidar.empty() && !c->imu.empty(); i++) {
            c->lidar.pop_front();
            c->imu.pop_front();
        }
    for (size_t i = 0; i + 1 < c->imu.size(); i++) c->imu[i].t -= lag;
    align_fronts_and_sizes(c->imu, c->lidar);
}

// LI_init.cpp:223-238
void cut_tail(li_calib* c) {
    for (int i = 0; i < 20 && !c->lidar.empty() && !c->imu.empty(); i++) {
        c->lidar.pop_back();
        c->imu.pop_back();
    }
    align_fronts_and_sizes(c->imu, c->lidar);
}

// One-direction 6th-order Butterworth low-pass (coefficients LI_init.h:219-225), LI_init.cpp:260-304.
const double kB[7] = {0.000076, 0.000457, 0.001143, 0.001524, 0.0011, 0.000457, 0.000076};
const double kA[7] = {1.0000, -4.182389, 7.491611, -7.313596, 4.089349, -1.238525, 0.158428};
constexpr int kTaps = 7, kExt = 10 * (kTaps - 1);

void butter(const Seq& in, Seq& out) {
    const int n = (int)in.size();
    // mirrored extension: in[60..1] | in[0..n-1] | in[n-2..n-61]
    std::vector<Sample> ext;
    ext.reserve(n + 2 * kExt);
    for (int k = kExt; k >= 1; k--) ext.push_back(in[k]);
    for (int k = 0; k < n; k++) ext.push_back(in[k]);
    for (int k = n - 2; k >= n - 1 - kExt; k--) ext.push_back(in[k]);
    std::vector<Sample> y(ext);
    const int m = (int)ext.size();
    for (int i = kTaps; i < m - kExt; i++) {
        V3 w, v, wa, va;
        for (int j = 0; j < kTaps; j++) {
            const Sample& s = ext[i - j];
            w = w + s.w * kB[j]; v = v + s.v * kB[j]; wa = wa + s.wa * kB[j]; va = va + s.va * kB[j];
        }
        for (int j = 1; j < kTaps; j++) {
            const Sample& s = y[i - j];
            w = w - s.w * kA[j]; v = v - s.v * kA[j]; wa = wa - s.wa * kA[j]; va = va - s.va * kA[j];
        }
        y[i].w = w; y[i].v = v; y[i].wa = wa; y[i].va = va;
    }
    for (int i = kExt; i < m - kExt; i++) out.push_back(y[i]);
}

// LI_init.cpp:306-315
void zero_phase(const Seq& in, Seq& out) {
    Seq f;
    butter(in, f);
    std::reverse(f.begin(), f.end());
    butter(f, out);
    std::reverse(out.begin(), out.end());
}

// LI_init.cpp:494-504
void normalize_acc(Seq& s) {
    V3 m;
    for (int i = 1; i < 10; i++) m = m + (s[i].va - m) / (double)i;
    const double nrm = m.norm();
    for (auto& e : s) e.va = e.va / nrm * kG;
}

// LI_init.cpp:160-193
void xcorr(li_calib* c, double odom_freq) {
    const int N = (int)c->imu.size();
    std::vector<double> a(N), b(N);
    double ma = 0, mb = 0;
    for (int i = 0; i < N; i++) {
        a[i] = c->imu[i].w.norm();
        b[i] = c->lidar[i].w.norm();
        ma += (a[i] - ma) / (i + 1);
        mb += (b[i] - mb) / (i + 1);
    }
    double best = -DBL_MAX;
    for (int lag = -N + 1; lag < N; lag++) {
        double corr = 0;
        const int i0 = std::max(0, -lag), i1 = std::min(N - 1, N - 1 - lag);
        for (int i = i0; i <= i1; i++) corr += (a[i] - ma) * (b[i + lag] - mb);
        if (corr > best) {
            best = corr;
            c->lag_frames = -lag;
        }
    }
    c->lag1 = c->lag_frames / odom_freq;
}

void push_row(std::vector<double>& v, std::initializer_list<double> r) { v.insert(v.end(), r); }

// LI_init.cpp:127-158
void central_diff(li_calib* c) {
    Seq& I = c->imu;
    Seq& L = c->lidar;
    for (int i = 1; i + 2 < (int)I.size(); i++) {
        double dt = I[i + 1].t - I[i - 1].t;
        I[i].wa = (I[i + 1].w - I[i - 1].w) / dt;
        push_row(c->log_rows[0], {I[i].w.x, I[i].w.y, I[i].w.z, I[i].w.norm(), I[i].va.x, I[i].va.y, I[i].va.z, I[i].wa.x, I[i].wa.y,
                                  I[i].wa.z, I[i].t});
    }
    for (int i = 1; i + 2 < (int)L.size(); i++) {
        double dt = L[i + 1].t - L[i - 1].t;
        L[i].wa = (L[i + 1].w - L[i - 1].w) / dt;
        L[i].va = (L[i + 1].v - L[i - 1].v) / dt;
        push_row(c->log_rows[1], {L[i].w.x, L[i].w.y, L[i].w.z, L[i].w.norm(), L[i].va.x, L[i].va.y, L[i].va.z + kG, L[i].wa.x, L[i].wa.y,
                                  L[i].wa.z, L[i].t});
    }
}

// LI_init.cpp:240-258
void acc_interpolate(li_calib* c) {
    Seq& I = c->imu;
    Seq& L = c->lidar;
    for (int i = 1; i + 1 < (int)L.size(); i++) {
        double d = L[i].t - I[i].t;
        if (d > 0) {
            double s = d / (I[i + 1].t - I[i].t);
            I[i].va = I[i + 1].va * s + I[i].va * (1 - s);
        } else {
            double s = -d / (I[i].t - I[i - 1].t);
            I[i].va = I[i - 1].va * s + I[i].va * (1 - s);
        }
        I[i].t += d;
    }
}

}  // namespace

extern "C" {

int li_calib_create(li_calib** out) {
    if (!out) return LI_CALIB_ERR_INVALID;
    *out = new li_calib();
    return LI_CALIB_OK;
}
void li_calib_destroy(li_calib* c) { delete c; }
void li_calib_set_data_accum_length(li_calib* c, double v) {
    if (c) c->data_accum_length = v;
}
void li_calib_set_solver(li_calib* c, int converge_fully) {
    if (c) c->solver = converge_fully ? 1 : 0;
}

int li_calib_push_imu_all(li_calib* c, const double omg[3], const double acc[3], double mean_acc_norm, double t) {
    if (!c || !omg || !acc || !(mean_acc_norm > 0)) return LI_CALIB_ERR_INVALID;
    Sample s;
    s.w = V3(omg[0], omg[1], omg[2]);
    s.va = V3(acc[0], acc[1], acc[2]) / mean_acc_norm * kG;
    s.t = t;
    c->imu_all.push_back(s);
    return LI_CALIB_OK;
}
int li_calib_push_lidar(li_calib* c, const double R[9], const double omg[3], const double vel[3], double t) {
    if (!c || !R || !omg || !vel) return LI_CALIB_ERR_INVALID;
    Sample s;
    std::memcpy(s.rot.m, R, sizeof s.rot.m);
    s.w = V3(omg[0], omg[1], omg[2]);
    s.v = V3(vel[0], vel[1], vel[2]);
    s.t = t;
    c->lidar.push_back(s);
    return LI_CALIB_OK;
}
int li_calib_push_imu(li_calib* c, const double omg[3], const double acc[3], double t) {
    if (!c || !omg || !acc) return LI_CALIB_ERR_INVALID;
    Sample s;
    s.w = V3(omg[0], omg[1], omg[2]);
    s.va = V3(acc[0], acc[1], acc[2]);
    s.t = t;
    c->imu.push_back(s);
    return LI_CALIB_OK;
}
int li_calib_sizes(const li_calib* c, int* a, int* i, int* l) {
    if (!c) return LI_CALIB_ERR_INVALID;
    if (a) *a = (int)c->imu_all.size();
    if (i) *i = (int)c->imu.size();
    if (l) *l = (int)c->lidar.size();
    return LI_CALIB_OK;
}
void li_calib_clear_imu_all(li_calib* c) {
    if (c) c->imu_all.clear();
}

int li_calib_data_sufficiency(li_calib* c, int frame_num, const double lidar_omg[3], int orig_odom_freq, int cut_frame_num,
                              double percent[3], int* sufficient) {
    if (!c || !lidar_omg || !sufficient || orig_odom_freq <= 0) return LI_CALIB_ERR_INVALID;
    M3 S = skew(V3(lidar_omg[0], lidar_omg[1], lidar_omg[2]));
    M3 StS = S.t() * S;
    for (int i = 0; i < 9; i++) c->hess_rot[i] += StS.m[i];
    *sufficient = 0;
    if (frame_num % orig_odom_freq * cut_frame_num == 0) {   // evaluated as (frame_num % freq) * cut, LI_init.cpp:515
        double w[3], V[9];
        eig_sym3(c->hess_rot, w, V);
        double s[3] = {w[0] / c->data_accum_length, w[1] / c->data_accum_length, w[2] / c->data_accum_length};
        double pr[3] = {s[1] * s[2], s[0] * s[2], s[0] * s[1]};
        if (percent) { percent[0] = pr[0]; percent[1] = pr[1]; percent[2] = pr[2]; }
        if (pr[0] > 0.99 && pr[1] > 0.99 && pr[2] > 0.99) *sufficient = 1;
    } else if (percent) {
        percent[0] = percent[1] = percent[2] = -1;
    }
    return LI_CALIB_OK;
}

int li_calib_initialize(li_calib* c, int orig_odom_freq, int cut_frame_num, double timediff_imu_wrt_lidar, double move_start_time,
                        int from_groups, li_calib_result* out) {
    if (!c || !out || orig_odom_freq <= 0 || cut_frame_num <= 0) return LI_CALIB_ERR_INVALID;
    for (auto& v : c->log_rows) v.clear();
    if (!from_groups) {
        if (c->imu_all.size() < 8 || c->lidar.empty()) return LI_CALIB_ERR_TOO_FEW;
        downsample_interpolate(c, move_start_time);
    }
    // fout_before_filter (:43-52, :592): the groups as they enter the filters, each without its last element
    for (size_t i = 0; i + 1 < c->imu.size(); i++) {
        const Sample& s = c->imu[i];
        push_row(c->log_rows[4], {s.w.x, s.w.y, s.w.z, s.w.norm(), s.va.x, s.va.y, s.va.z, s.t});
    }
    for (size_t i = 0; i + 1 < c->lidar.size(); i++) {
        const Sample& s = c->lidar[i];
        push_row(c->log_rows[5], {s.w.x, s.w.y, s.w.z, s.w.norm(), s.t});
    }
    const size_t need = 2 * kExt + 2 + 10 + 20 + 8;
    if (c->imu.size() < need || c->lidar.size() < need) return LI_CALIB_ERR_TOO_FEW;
    time_compensate(c, 0.0, true);                                       // :592
    if (c->imu.size() < 2 * kExt + 24) return LI_CALIB_ERR_TOO_FEW;

    {   // first zero-phase pass (:595-601); set_IMU_state / set_Lidar_state drop the last element (:27-33)
        Seq fi, fl;
        zero_phase(c->imu, fi);
        normalize_acc(fi);
        zero_phase(c->lidar, fl);
        fi.pop_back();
        fl.pop_back();
        c->imu.swap(fi);
        c->lidar.swap(fl);
    }
    cut_tail(c);                                                          // :602
    if (c->imu.size() < 2 * kExt + 4) return LI_CALIB_ERR_TOO_FEW;
    xcorr(c, (double)(orig_odom_freq * cut_frame_num));                   // :604
    time_compensate(c, c->lag1, false);                                   // :605
    if (c->imu.size() < 2 * kExt + 4) return LI_CALIB_ERR_TOO_FEW;
    central_diff(c);                                                      // :607
    {   // second zero-phase pass: only the derivatives are taken over (:35-41, :609-613)
        Seq fi, fl;
        zero_phase(c->imu, fi);
        zero_phase(c->lidar, fl);
        for (size_t i = 0; i < c->imu.size(); i++) {
            c->imu[i].wa = fi[i].wa;
            c->lidar[i].wa = fl[i].wa;
            c->lidar[i].va = fl[i].va;
        }
    }

    // solve_Rotation_only (:317-343)
    RotOnly p1;
    p1.I = &c->imu; p1.L = &c->lidar;
    M3 R;
    Quat q;                                  // R_LI_quat = (1,0,0,0), :318-322
    if (c->solver == 0) {
        out->iters_rot = tr_solve_reference_schedule(p1, q, nullptr, &out->cost_rot);
        R = quat_to_rot(q);
    } else {
        out->iters_rot = lm_solve(p1, R, nullptr, &out->cost_rot);
    }
    c->R_LI = R;

    // solve_Rot_bias_gyro (:345-401)
    RotBias p2;
    p2.np = 4;
    for (int k = 0; k < 4; k++) { p2.lo[k] = -INFINITY; p2.hi[k] = INFINITY; }
    p2.I = &c->imu; p2.L = &c->lidar;
    double q2[4] = {0, 0, 0, 0};
    if (c->solver == 0) {
        // the reference re-seeds the quaternion from the rotation matrix (Eigen::Quaterniond quat(Rot_Lidar_wrt_IMU), :346):
        // q is unit up to rounding, the matrix round trip changes nothing beyond that
        out->iters_rot_bias = tr_solve_reference_schedule(p2, q, q2, &out->cost_rot_bias);
        R = quat_to_rot(q);
    } else {
        out->iters_rot_bias = lm_solve(p2, R, q2, &out->cost_rot_bias);
    }
    c->R_LI = R;
    c->bg = V3(q2[0], q2[1], q2[2]);
    c->lag2 = q2[3];
    c->total_lag = c->lag1 + c->lag2;
    time_compensate(c, c->lag2, false);
    for (size_t i = 0; i < c->lidar.size(); i++) {
        V3 v = c->R_LI * c->lidar[i].w + c->bg;
        push_row(c->log_rows[2], {v.x, v.y, v.z, c->lidar[i].t});
    }

    acc_interpolate(c);                                                   // :619

    // solve_trans_biasacc_grav (:403-492)
    TransAcc p3;
    p3.np = 6;
    for (int k = 0; k < 3; k++) { p3.lo[k] = -0.01; p3.hi[k] = 0.01; }   // :448-451
    for (int k = 3; k < 6; k++) { p3.lo[k] = -INFINITY; p3.hi[k] = INFINITY; }
    p3.I = &c->imu; p3.L = &c->lidar; p3.R_LI = c->R_LI;
    M3 RG;
    double q3[6] = {0, 0, 0, 0, 0, 0};
    if (c->solver == 0) {
        // bounded problem: Ceres additionally line-searches along the projected step; here the candidate is the
        // projection itself (the schedule and the stopping rule are the same)
        Quat qg;
        out->iters_trans = tr_solve_reference_schedule(p3, qg, q3, &out->cost_trans);
        RG = quat_to_rot(qg);
    } else {
        out->iters_trans = lm_solve(p3, RG, q3, &out->cost_trans);
    }
    c->R_GL0 = RG;
    c->grav_L0 = RG * V3(0, 0, -kG);
    V3 baL(q3[0], q3[1], q3[2]), TIL(q3[3], q3[4], q3[5]);
    c->ba = c->R_LI * baL;
    c->T_LI = (c->R_LI * TIL) * -1.0;
    {
        M3 RLIt = c->R_LI.t();
        for (size_t i = 0; i < c->imu.size(); i++) {
            const Sample& l = c->lidar[i];
            M3 Wx = skew(l.w);
            M3 Mi = madd(Wx * Wx, skew(l.wa));
            V3 aI = l.rot * (RLIt * c->imu[i].va) - l.rot * baL;
            V3 aL = l.va + l.rot * (Mi * TIL) - c->grav_L0;
            push_row(c->log_rows[3], {aI.x, aI.y, aI.z, aL.x, aL.y, aL.z, c->imu[i].t, l.t});
        }
    }

    std::memcpy(out->R_LI, c->R_LI.m, sizeof out->R_LI);
    out->T_LI[0] = c->T_LI.x; out->T_LI[1] = c->T_LI.y; out->T_LI[2] = c->T_LI.z;
    out->gyro_bias[0] = c->bg.x; out->gyro_bias[1] = c->bg.y; out->gyro_bias[2] = c->bg.z;
    out->acc_bias[0] = c->ba.x; out->acc_bias[1] = c->ba.y; out->acc_bias[2] = c->ba.z;
    out->grav_L0[0] = c->grav_L0.x; out->grav_L0[1] = c->grav_L0.y; out->grav_L0[2] = c->grav_L0.z;
    out->time_lag_1 = c->lag1;
    out->time_lag_2 = c->lag2;
    out->time_L_I = timediff_imu_wrt_lidar + c->total_lag;
    V3 e = rot_to_euler(c->R_LI);
    out->euler_deg[0] = e.x * 57.3; out->euler_deg[1] = e.y * 57.3; out->euler_deg[2] = e.z * 57.3;
    out->lag_frames = c->lag_frames;
    out->n_samples = (int)c->imu.size();
    return LI_CALIB_OK;
}

int li_calib_log_rows(const li_calib* c, int which, double* out, int cap_rows, int* rows) {
    if (!c || which < 0 || which > 5 || !rows) return LI_CALIB_ERR_INVALID;
    static const int cols[6] = {11, 11, 4, 8, 8, 5};
    const std::vector<double>& v = c->log_rows[which];
    const int n = (int)(v.size() / cols[which]);
    *rows = n;
    if (out && cap_rows > 0) std::memcpy(out, v.data(), sizeof(double) * cols[which] * (size_t)std::min(n, cap_rows));
    return LI_CALIB_OK;
}

}  // extern "C"
