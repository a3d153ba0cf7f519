/* liinit_calib.h -- C-ABI of the LI-Init batch initialisation (SURVEY.md section 8f, row N4): the temporal + spatial
 * LiDAR-IMU calibration the node runs once the odometry of the hot path has gathered enough excitation
 * (reference: include/LI_init/LI_init.h:91-357, include/LI_init/LI_init.cpp:9-650; driven from
 * src/laserMapping.cpp:428-430, :1190-1217). Host only: the whole stage handles ~1.4k samples once per run, there is
 * nothing for a GPU in it. It is restated without Ceres / Eigen (neither is installed here): the three non-linear
 * least-squares problems are solved by an own trust-region Levenberg-Marquardt on SO(3) x R^n (see li_calib_set_solver).
 *
 * Plain C: doubles, row-major 3x3 matrices, no ROS / Eigen types.
 */
#ifndef LIINIT_CALIB_H
#define LIINIT_CALIB_H

#ifdef __cplusplus
extern "C" {
#endif

typedef struct li_calib li_calib;

#define LI_CALIB_OK 0
#define LI_CALIB_ERR_INVALID (-1)
#define LI_CALIB_ERR_TOO_FEW (-2) /* fewer samples than the filter extension needs (LI_init.cpp:261-274: 2*60+1) */

/* What LI_Initialization leaves in the LI_Init object (LI_init.h:335-347) and prints (LI_init.cpp:634-650). */
typedef struct li_calib_result {
    double R_LI[9];        /* Rot_Lidar_wrt_IMU   (get_R_LI) */
    double T_LI[3];        /* Trans_Lidar_wrt_IMU (get_T_LI) */
    double gyro_bias[3];   /* get_gyro_bias */
    double acc_bias[3];    /* get_acc_bias (IMU frame) */
    double grav_L0[3];     /* get_Grav_L0: gravity in the first LiDAR frame */
    double time_lag_1;     /* cross-correlation lag / odom_freq (LI_init.cpp:160-193) */
    double time_lag_2;     /* lag from the unified optimisation (:345-401) */
    double time_L_I;       /* timediff_imu_wrt_lidar + time_lag_1 + time_lag_2, the printed "Time Lag IMU to LiDAR" (:625) */
    double euler_deg[3];   /* RotMtoEuler(R_LI) * 57.3, as printed (:639) */
    int lag_frames;        /* lag_IMU_wtr_Lidar */
    int n_samples;         /* aligned sample pairs entering the three solves */
    int iters_rot, iters_rot_bias, iters_trans; /* LM iterations of the three problems */
    double cost_rot, cost_rot_bias, cost_trans; /* 0.5 * sum of squared residuals at the solution */
} li_calib_result;

/* LI_Init::LI_Init (LI_init.cpp:9-24). */
int li_calib_create(li_calib** out);
void li_calib_destroy(li_calib* c);
/* data_accum_length (LI_init.cpp:17, launch parameter initialization/data_accum_length, laserMapping.cpp:790). */
void li_calib_set_data_accum_length(li_calib* c, double v);
/* 0 (default): the three solves follow the schedule and stopping rule of ceres::Solve with default options, as the
 * reference calls it (LI_init.cpp:336-339,:383-385,:453-455) -- stops, like the reference, a few 1e-5 short of the
 * optimum and so reproduces its numbers. 1: Levenberg-Marquardt run to convergence (the exact least-squares optimum). */
void li_calib_set_solver(li_calib* c, int converge_fully);

/* push_ALL_IMU_CalibState (LI_init.cpp:54-62): every IMU message while LiDAR-only odometry runs; acc is rescaled by
 * G_m_s2 / mean_acc_norm. */
int li_calib_push_imu_all(li_calib* c, const double omg[3], const double acc[3], double mean_acc_norm, double t);
/* push_Lidar_CalibState (:72-80): per scan, the odometry's rotation, angular velocity (state.bias_g in LO mode),
 * linear velocity and the scan end time (laserMapping.cpp:1192). */
int li_calib_push_lidar(li_calib* c, const double R[9], const double omg[3], const double vel[3], double t);
/* push_IMU_CalibState (:64-70): an IMU sample already interpolated to a LiDAR time stamp. Together with
 * li_calib_push_lidar this loads the state groups as they are right after downsample_interpolate_IMU, which is what
 * the reference dumps to Log/IMU_before_filter.txt / Log/Lidar_before_filter.txt (:43-52) -- the replay entry. */
int li_calib_push_imu(li_calib* c, const double omg[3], const double acc[3], double t);
int li_calib_sizes(const li_calib* c, int* n_imu_all, int* n_imu, int* n_lidar);
void li_calib_clear_imu_all(li_calib* c); /* IMU_buffer_clear (LI_init.h:288-290) */

/* data_sufficiency_assess (:506-563): adds the frame's rotation Jacobian, and once per second of odometry evaluates
 * the excitation. percent[3] = Rot_percent (x, y, z of the eigen basis, unclamped), *sufficient as the return value of
 * the reference. The progress bars are not drawn. */
int li_calib_data_sufficiency(li_calib* c, int frame_num, const double lidar_omg[3], int orig_odom_freq, int cut_frame_num,
                              double percent[3], int* sufficient);

/* LI_Initialization (:586-632). from_groups != 0 skips downsample_interpolate_IMU (the groups were loaded with
 * li_calib_push_imu / li_calib_push_lidar). */
int li_calib_initialize(li_calib* c, int orig_odom_freq, int cut_frame_num, double timediff_imu_wrt_lidar, double move_start_time,
                        int from_groups, li_calib_result* out);

/* The rows the reference writes to Log/ during LI_Initialization, for replay checks:
 *   0: IMU_meas.txt    (:135-139)  ang_vel(3) |ang_vel| linear_acc(3) ang_acc(3) t            -> 11 columns
 *   1: LiDAR_meas.txt  (:151-157)  ang_vel(3) |ang_vel| linear_acc-STD_GRAV(3) ang_acc(3) t   -> 11 columns
 *   2: Lidar_omg_after_rot.txt (:397-400)  R_LI*ang_vel + gyro_bias (3) t                      ->  4 columns
 *   3: acc_cost.txt    (:477-484)  acc_I(3) acc_L(3) t_IMU t_LiDAR                             ->  8 columns
 *   4: IMU_before_filter.txt   (:43-47)  ang_vel(3) |ang_vel| linear_acc(3) t                  ->  8 columns
 *   5: Lidar_before_filter.txt (:48-51)  ang_vel(3) |ang_vel| t                                ->  5 columns
 * Tables 4 and 5 are the IMU / LiDAR groups entering the filters (after downsample_interpolate_IMU, or as loaded with
 * from_groups), each without its last element, as fout_before_filter writes them.
 * out: row-major [cap_rows x columns]; *rows = rows available. */
int li_calib_log_rows(const li_calib* c, int which, double* out, int cap_rows, int* rows);

#ifdef __cplusplus
}
#endif
#endif
