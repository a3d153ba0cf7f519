/* liinit_host.h -- host side of the drop-in: the part of laserMapping.cpp:936-1134 that the north star keeps on
 * the CPU (IESKF solve, state update, convergence / rematch policy, covariance update), re-expressed over the
 * C-ABI of include/liinit_gpu.h so that only HtH (12x12), Htr (12) and m cross the PCIe bus per iteration
 * (SURVEY.md 8a row A8). Plain C++17, no Eigen/PCL/ROS (none is installed here); see INTEGRATION.md for the
 * Eigen-typed call sites in the node.
 */
#ifndef LIINIT_HOST_H
#define LIINIT_HOST_H

#include "liinit_gpu.h"

#ifdef __cplusplus
extern "C" {
#endif

#define LIINIT_DIM_STATE 24 /* include/common_lib.h:24 */

/* StatesGroup (include/common_lib.h:68-169), flat, row-major. State vector order for boxplus / boxminus:
 * [rot 0:3 | pos 3:6 | R_LI 6:9 | T_LI 9:12 | vel 12:15 | bg 15:18 | ba 18:21 | g 21:24]. */
typedef struct liinit_state {
    double rot_end[9];
    double pos_end[3];
    double offset_R_L_I[9];
    double offset_T_L_I[3];
    double vel_end[3];
    double bias_g[3];
    double bias_a[3];
    double gravity[3];
    double cov[LIINIT_DIM_STATE * LIINIT_DIM_STATE];
} liinit_state;

typedef struct liinit_scan_stats {
    int iterations;        /* passes run (<= max_iteration) */
    int search_passes;     /* of which nearest_search_en was true */
    int effect_feat_num;   /* m of the last pass */
    int converged;         /* flg_EKF_converged of the last pass */
    double last_rot_deg;   /* deltaR, laserMapping.cpp:1096 */
    double last_trans_cm;  /* deltaT, :1097 */
    double res_sq;         /* sum of pd2^2 over the selected points of the last pass */
} liinit_scan_stats;

/* StatesGroup() defaults (common_lib.h:70-81): identity rotations, zero vectors, cov = I with [15:24] = 1e-5. */
void liinit_state_init(liinit_state* s);
/* operator+= (common_lib.h:124-135) and operator- (:137-151). */
void liinit_state_boxplus(liinit_state* s, const double delta[LIINIT_DIM_STATE]);
void liinit_state_boxminus(const liinit_state* a, const liinit_state* b, double out[LIINIT_DIM_STATE]);
/* Exp(v1,v2,v3) (so3_math.h:61-80) and Log(R) (:100-107). */
void liinit_so3_exp(const double v[3], double R[9]);
void liinit_so3_log(const double R[9], double v[3]);

/* One IESKF update from the device accumulators: the information-form equivalent of laserMapping.cpp:1080-1087.
 *   K_1 = (blkdiag(1000*HtH, 0) + cov^-1)^-1 ; solution = K_1[:,0:12]*(1000*Htr) + vec - K_1[:,0:12]*(1000*HtH)*vec[0:12],
 *   vec = state_propagat (-) state ; state (+)= solution.  KH (24x12, may be NULL) = K_1[:,0:12]*(1000*HtH) = K*Hsub (:1113). */
int liinit_ieskf_update(liinit_state* state, const liinit_state* state_propagat, const double HtH[144], const double Htr[12],
                        double solution[LIINIT_DIM_STATE], double* KH);

/* The whole per-scan update, laserMapping.cpp:936-1134, on an uploaded scan (liinit_scan_upload): iterates
 * liinit_icp_iterate + liinit_ieskf_update with the reference's rematch / convergence policy and covariance update.
 * state: in = propagated prior (state_propagat = state, :910), out = posterior. */
int liinit_scan_update(liinit_ctx* h, liinit_state* state, int max_iteration, int imu_en, liinit_scan_stats* stats);

/* liinit_ieskf_update and liinit_scan_update with the extrinsic (offset_R_L_I, offset_T_L_I: states 6:12) held constant, for a replay
 * of the LIO phase with a candidate calibration. The update solves on the other 18 states: cov restricted to them is inverted, only the
 * pose block HtH[0:6, 0:6] / Htr[0:6] of the 12-column Jacobian enters, and solution[6:12] = 0. The extrinsic is left bit for bit as it
 * was, and on return its rows and columns of cov are zero (so are those of KH). With the extrinsic's propagation noise set to zero
 * (liinit_imu_set_R_LI_cov / _T_LI_cov), liinit_imu_propagate keeps them zero. */
int liinit_ieskf_update_frozen(liinit_state* state, const liinit_state* state_propagat, const double HtH[144], const double Htr[12],
                               double solution[LIINIT_DIM_STATE], double* KH);
int liinit_scan_update_frozen(liinit_ctx* h, liinit_state* state, int max_iteration, int imu_en, liinit_scan_stats* stats);

/* State propagation of the LiDAR-only (constant-velocity) mode, ImuProcess::Forward_propagation_without_imu without its
 * point loop (src/IMU_Processing.hpp:212-243; the loop :246-266 is liinit_raw_undistort_cv): bias_g stands for the
 * angular velocity, vel_end for the linear velocity. cov <- F cov F^T + Q with F[0:3,0:3] = Exp(-bias_g dt),
 * F[0:3,15:18] = F[3:6,12:15] = I dt, Q[15:18] = cov_gyr_scale dt^2, Q[12:15] = cov_acc_scale dt^2; then
 * rot_end <- rot_end Exp(bias_g dt), pos_end += vel_end dt. dt: scan-to-scan time (0.1 for the first frame, :217-223). */
void liinit_propagate_cv(liinit_state* s, double dt, const double cov_gyr_scale[3], const double cov_acc_scale[3]);

/* ---- the IMU branch of ImuProcess (src/IMU_Processing.hpp), used in LIO mode after the hand-over of LI_Initialization ---- */
#define LIINIT_IMU_SAMPLE_DOUBLES 7   /* one IMU sample: {stamp [s], gyr xyz [rad/s], acc xyz} */
#define LIINIT_POSE6D_DOUBLES 22      /* Pose6D (common_lib.h:184-199): {offset_time, acc[3], gyr[3], vel[3], pos[3], rot[9]} */

/* The members of ImuProcess (IMU_Processing.hpp:56-89) that its IMU branch reads or writes. */
typedef struct liinit_imu {
    double last_imu[LIINIT_IMU_SAMPLE_DOUBLES];   /* last_imu_: last sample of the previous measure group */
    double angvel_last[3];        /* bias-corrected mean angular velocity of the last IMU interval */
    double acc_s_last[3];         /* world-frame acceleration of the last IMU interval */
    double last_lidar_end_time;   /* last_lidar_end_time_: end of the previous scan */
    double cov_acc[3];
    double cov_gyr[3];
    double cov_acc_scale[3];
    double cov_gyr_scale[3];
    double cov_R_LI[3];
    double cov_T_LI[3];
    double cov_bias_gyr[3];
    double cov_bias_acc[3];
    double mean_acc_norm;         /* IMU_mean_acc_norm: the accelerometer reading of 1 g */
    int need_init;                /* imu_need_init_ */
    int reserved;
} liinit_imu;

/* ImuProcess() (IMU_Processing.hpp:92-108): cov_acc = cov_gyr = 0.1, cov_R_LI = 1e-5, cov_T_LI = 1e-4, bias covariances 1e-4,
 * angvel_last = 0, last_imu_ = a zero sample, need_init = 1. Members the constructor leaves unset get the values the node sets
 * before first use: cov_acc_scale = cov_gyr_scale = 0.1 and mean_acc_norm = 9.81 (laserMapping.cpp:76,94). acc_s_last and
 * last_lidar_end_time, never written before the first propagation in LI-Init, are 0. */
void liinit_imu_init(liinit_imu* imu);
/* The setters the node calls (laserMapping.cpp:833-838 from the YAML, :1224-1228 at the hand-over). set_gyr_cov / set_acc_cov
 * set the scales (cov_gyr_scale / cov_acc_scale), as the reference's do. */
void liinit_imu_set_gyr_cov(liinit_imu* imu, const double v[3]);
void liinit_imu_set_acc_cov(liinit_imu* imu, const double v[3]);
void liinit_imu_set_R_LI_cov(liinit_imu* imu, const double v[3]);
void liinit_imu_set_T_LI_cov(liinit_imu* imu, const double v[3]);
void liinit_imu_set_gyr_bias_cov(liinit_imu* imu, const double v[3]);
void liinit_imu_set_acc_bias_cov(liinit_imu* imu, const double v[3]);
void liinit_imu_set_mean_acc_norm(liinit_imu* imu, double mean_acc_norm);

/* The switch scan, the first scan after LI_init_done (Process, IMU_Processing.hpp:445-453): records the last of the n samples as
 * last_imu_, sets cov_acc / cov_gyr from the scales and clears need_init. Nothing is propagated and the state is not an argument:
 * the scan reuses the previous undistorted cloud (Process returns before touching it). n = 0: nothing happens (:423). */
int liinit_imu_switch(liinit_imu* imu, const double* samples, int n);

/* The forward part of propagation_and_undist (IMU_Processing.hpp:271-382) for one measure group of n samples
 * (n x LIINIT_IMU_SAMPLE_DOUBLES, ascending stamps): last_imu_ is put in front, pairs whose later sample is older than
 * last_lidar_end_time are skipped, each remaining pair propagates the state (mean rate minus bias_g, mean specific force scaled
 * by 9.81 / mean_acc_norm minus bias_a) and the covariance (cov <- F cov F^T + Q), then the state is extrapolated to the scan end
 * pcl_beg_time + pcl_end_offset_ms / 1000 (forwards or backwards, :374-378).
 * poses: the IMUpose table for liinit_raw_undistort_imu, room for n + 1 poses of LIINIT_POSE6D_DOUBLES; *npose its length.
 * n = 0: nothing happens, *npose = 0 (Process returns at once, :423). LIINIT_ERR_INVALID while need_init is set (the switch scan
 * comes first); LIINIT_ERR_CAPACITY, with nothing changed, when the table would be longer than LIINIT_MAX_IMU_POSES. */
int liinit_imu_propagate(liinit_imu* imu, liinit_state* s, const double* samples, int n, double pcl_beg_time, double pcl_end_offset_ms,
                         double* poses, int* npose);

/* ---- the LIO phase of a replay (DESIGN.md section 4d), natively: assess.Replay.run after the hand-over with no Python in between ----
 * The hand-over itself (the candidate extrinsic and lag, and for a frozen replay the zero extrinsic rows / columns of cov and the zero
 * extrinsic noise of the IMU processor) is the caller's; the job holds what the loop starts from. Each event is either a stored
 * sub-frame (its index in the replay store, liinit_replay_*) or LIINIT_REPLAY_IMU, the next of the recorded IMU samples. The loop:
 *   an IMU sample: imu_cbk's compensation (stamp = t - timediff - time_lag; an older stamp than the last clears the buffer), appended;
 *   a sub-frame: queued; then, while the oldest queued sub-frame's lidar_end_time = t_beg + end_ms / 1000 has an IMU stamp at or after
 *   it (sync_packages), its measure group is popped and process_raw's LIO body runs: a group with the IMU processor switched propagates
 *   (liinit_imu_propagate), stages the sub-frame (liinit_replay_stage) and undistorts it (liinit_raw_undistort_imu, two poses or more);
 *   a group before the switch switches it (liinit_imu_switch: the switch scan); an empty group does neither. Then liinit_raw_downsample
 *   (filter_size_surf as float), liinit_scan_update[_frozen] (imu_en), liinit_map_incremental (filter_size_map) and, for every update but
 *   the switch scan, liinit_assess_append of the staged cloud with the posterior pose and extrinsic.
 * The map must be ready (the hand-over comes after the LiDAR-only phase built it): the loop never builds one. */
#define LIINIT_REPLAY_IMU (-1)
typedef struct liinit_replay_job {
    liinit_state state;           /* the state after the hand-over */
    liinit_imu imu;               /* the IMU processor after the hand-over */
    const double* buf_rows;       /* the IMU buffer after the hand-over: n_buf rows {stamp, gyr xyz, acc xyz}, stamps compensated */
    const double* samples;        /* the recorded IMU samples as they arrived, n_samples x {t, gyr xyz, acc xyz} */
    const int* events;            /* n_events: a stored sub-frame index (>= 0) or LIINIT_REPLAY_IMU */
    double last_stamp;            /* the buffer's last compensated stamp (-inf: none) */
    double timediff;              /* timediff_imu_wrt_lidar */
    double time_lag;              /* time_lag_IMU_wtr_lidar, the candidate's */
    double filter_size_surf;      /* the scan voxel grid's leaf */
    double filter_size_map;       /* map_incremental's ds */
    int n_buf, n_samples, n_events;
    int frame_num;                /* the loop's frame counter at the hand-over */
    int switch_scan;              /* frame_num of the switch scan; -1: not yet */
    int max_iteration;
    int frozen;                   /* liinit_scan_update_frozen: the extrinsic held constant */
    int reserved;
} liinit_replay_job;
/* Runs the loop on h. states[k] / frames[k] (room for cap): the posterior state and the stored sub-frame index of update k, for
 * *n_updates updates. Returns LIINIT_OK, or the code of the first call that failed (the updates before it are in states / frames);
 * LIINIT_ERR_INVALID for a bad job (an event past the recorded samples, a negative count), LIINIT_ERR_CAPACITY when cap is too small. */
int liinit_replay_run(liinit_ctx* h, const liinit_replay_job* job, liinit_state* states, int* frames, int cap, int* n_updates);

/* lasermap_fov_segment (laserMapping.cpp:260-305): keeps a cube_len-sized local map box around the LiDAR and, when the
 * LiDAR comes within MOV_THRESHOLD*det_range of a face, shifts the box and returns the slabs that fell out of it
 * (cub_needrm) -- the boxes to hand to liinit_map_delete_boxes. local_box: {min xyz, max xyz}, state kept by the caller;
 * *initialized: Localmap_Initialized. boxes_out: room for 3 boxes (18 floats). Returns the number of boxes (0..3). */
int liinit_fov_segment(const double pos_LiD[3], double cube_len, double det_range, float local_box[6], int* initialized,
                       float boxes_out[18]);

#ifdef __cplusplus
}
#endif
#endif
