/* include/liinit_gpu.h -- C-ABI of the CUDA-native (H100, sm_90a) ICP measurement model of LI-Init.
 *
 * The reference has NO plugin / FFI boundary on this path: the code is inlined in
 * main() over file-scope globals (/root/reference/src/laserMapping.cpp:102-125,
 * 957-1134) and the only real API on it is the C++ class KD_TREE
 * (include/ikd-Tree/ikd_Tree.h:165-187). This header is the cut SURVEY.md section 8(b)
 * introduces; every entry point cites the reference lines it replaces.
 *
 * Conventions: extern "C"; opaque context; int return codes (0 = LIINIT_OK, <0 =
 * error, message via liinit_last_error); no exceptions cross the ABI; the caller
 * owns every host buffer, the library owns all device memory; one thread at a time
 * per context (the node drives its one context from its main thread,
 * laserMapping.cpp:891-1238); distinct contexts may be driven from distinct threads
 * at once. Each context is internally asynchronous on its own non-blocking CUDA
 * stream. (What makes that safe: the library keeps no process-wide state on any
 * path but liinit_create's error text, which is thread_local, and the lazy dlopen of
 * NCCL behind liinit_comm_*; the host library, liinit_host.h, keeps none at all.
 * A call that names two contexts -- liinit_replay_share -- counts as a call on
 * both.) Matrices are row-major doubles. Point arrays are float with a
 * caller-given stride in floats: 3 (packed xyz), 4 (float4) or 12 (the 48-byte
 * pcl::PointXYZINormal of include/common_lib.h:37 -- x,y,z are its first floats).
 *
 * There is NO CPU fallback: every compute entry point fails with
 * LIINIT_ERR_CUDA when no sm_90-class device is usable.
 */
#ifndef LIINIT_GPU_H
#define LIINIT_GPU_H

#ifdef __cplusplus
extern "C" {
#endif

#define LIINIT_OK 0
#define LIINIT_ERR_INVALID (-1)   /* bad argument / call order */
#define LIINIT_ERR_CUDA (-2)      /* CUDA runtime error (no device, launch failure, ...) */
#define LIINIT_ERR_CAPACITY (-3)  /* map / scan / hash capacity exceeded */

#define LIINIT_NUM_MATCH_POINTS 5 /* include/common_lib.h:28 */

#define LIINIT_KNN_BRICKS 1
#define LIINIT_KNN_CELLS 2
/* (3, 4, 5 were the hybrid, TMA-fused and warp-per-point searches of round 2: measured slower, removed) */

typedef struct liinit_ctx liinit_ctx;

typedef struct liinit_config {
    float filter_size_map;   /* mapping/filter_size_map (config/avia.yaml:23): map voxel ds; KD_TREE::set_downsample_param (laserMapping.cpp:923) */
    int max_map_points;      /* capacity of the device map (live points); e.g. 50M for BASELINE config 4 */
    int max_scan_points;     /* capacity per scan (replaces the fixed 100000 caps, laserMapping.cpp:108-109,117-119) */
    int device_id;           /* CUDA device ordinal */
    int brick_cells_log2;    /* voxels per brick edge = 1<<this; 0 -> default (3, i.e. brick edge = 8*ds) */
    int hash_capacity_log2;  /* brick hash slots = 1<<this; 0 -> derived from max_map_points */
    int knn_group_lanes;     /* lanes cooperating on one scan point in the lockstep 5-NN kernel: 2, 4, 8, 16 or 32; 0 -> chosen per pass from the frame
                                size (32 lanes up to 14k points, 8 up to 70k, 4 beyond: small frames need the latency, large ones the throughput) */
    float knn_seed_radius_cells; /* first search shell of the 5-NN kernel, in map voxels (radius = this * filter_size_map); 0 -> default (2) */
    int knn_index;           /* how the 5-NN kernel searches the brick hash: LIINIT_KNN_BRICKS (lockstep groups of knn_group_lanes lanes over whole bricks)
                                or LIINIT_KNN_CELLS (thread per scan point over the per-brick cell directory; needs brick_cells_log2 = 3); 0 -> default */
    int reserved[6];
} liinit_config;

/* lifecycle ------------------------------------------------------------------ */
int liinit_create(const liinit_config* cfg, liinit_ctx** out);
int liinit_destroy(liinit_ctx* h);
const char* liinit_last_error(const liinit_ctx* h);   /* h may be NULL: error of the last failed liinit_create */
/* Run on an externally owned stream (cudaStream_t as void*); NULL -> the context's own stream. */
int liinit_set_stream(liinit_ctx* h, void* cuda_stream);

/* map (replaces KD_TREE, include/ikd-Tree/ikd_Tree.h:165-187) ------------------ */
/* KD_TREE::Build (ikd_Tree.cpp:336-347; call site laserMapping.cpp:921-928): replaces the map, no downsampling. */
int liinit_map_build(liinit_ctx* h, const float* xyz, int stride_floats, int n);
/* KD_TREE::Add_Points(points, downsample_on) (ikd_Tree.cpp:381-456; call sites laserMapping.cpp:556-557).
 * added: number of voxels whose content changed (downsample_on) / points appended. */
int liinit_map_add_points(liinit_ctx* h, const float* xyz, int stride_floats, int n, int downsample_on, int* added);
/* KD_TREE::Delete_Point_Boxes (ikd_Tree.cpp:500-520; SURVEY.md row N1 -- the node computes cub_needrm at
 * laserMapping.cpp:260-305 but never passes it on). boxes: nbox x {min x,y,z, max x,y,z} (BoxPointType, ikd_Tree.h:63-66);
 * a point is deleted iff min <= p < max on every axis (:633). deleted: number of points removed. */
int liinit_map_delete_boxes(liinit_ctx* h, const float* boxes, int nbox, int* deleted);
/* Housekeeping the kd-tree does by rebuilding (ikd_Tree.cpp:586-606): slabs abandoned by growth and points removed by box deletes
 * are given back -- live points are re-inserted into a cleared pool, empty bricks leave the hash. Called automatically by
 * liinit_map_add_points / liinit_map_incremental when the pool allocator is in its last quarter and at least half of it is dead;
 * the live set is unchanged. */
int liinit_map_compact(liinit_ctx* h);
/* KD_TREE::validnum / size (ikd_Tree.cpp:71-88,120-137; laserMapping.cpp:932-933,1142): live points. */
int liinit_map_validnum(liinit_ctx* h, int* n);
int liinit_map_size(liinit_ctx* h, int* n);
/* KD_TREE::flatten(Root_Node, out, NOT_RECORD) (ikd_Tree.cpp:1229-1255; laserMapping.cpp:251): live points, packed xyz. */
int liinit_map_download(liinit_ctx* h, float* xyz, int cap_points, int* n);
/* KD_TREE::Nearest_Search for n arbitrary world-frame queries (ikd_Tree.cpp:349-379), max_dist as at laserMapping.cpp:980:
 * squared distance <= max_dist (sic). k must be 5. out_xyz [n*5*3], out_d2 [n*5] (-1 where missing), out_cnt [n]. */
int liinit_map_nearest_search(liinit_ctx* h, const float* q_xyz, int stride_floats, int n, double max_dist,
                              float* out_xyz, float* out_d2, int* out_cnt);

/* per-scan hot path (replaces laserMapping.cpp:936-1080) ---------------------------- */
/* feats_down_body (laserMapping.cpp:917-919): once per scan; resets selection flags / neighbour lists. */
int liinit_scan_upload(liinit_ctx* h, const float* body_xyz, int stride_floats, int n);
/* Same role, without the staging copy: body_xyz must be page-locked host memory the device can address (cudaHostAlloc,
 * cudaHostRegister, a pinned torch tensor). Nothing is transferred by this call: the search kernel of the next
 * liinit_icp_iterate pass reads the coordinates over PCIe itself and leaves the packed copy in HBM for the later
 * passes of the scan (any other consumer triggers the copy first). The buffer must stay valid and unmodified until
 * that first pass (or liinit_scan_update / liinit_map_incremental / liinit_scan_download_body) has returned; with
 * liinit_icp_iterate_device, until the work queued on the stream has completed.
 * LIINIT_ERR_INVALID when the pointer is not device-addressable page-locked memory. */
int liinit_scan_attach_host(liinit_ctx* h, const float* pinned_body_xyz, int stride_floats, int n);
/* ---- raw-scan front end (SURVEY.md section 8f rows N3, N2): raw points -> undistort -> voxel grid -> resident scan ---- */
/* Stage a raw cloud on the device. time_index: float index of the per-point time offset in MILLISECONDS inside a point
 * (9 = PointType.curvature, src/preprocess.cpp), or -1 when there is none. */
int liinit_raw_upload(liinit_ctx* h, const float* pts, int stride_floats, int time_index, int n);
/* Forward_propagation_without_imu's un-distortion loop (IMU_Processing.hpp:246-266; constant-velocity model, LO mode):
 * omega = state.bias_g (angular velocity), rot_end / vel_end = the PROPAGATED state. In place on the staged cloud. */
int liinit_raw_undistort_cv(liinit_ctx* h, const double omega[3], const double rot_end[9], const double vel_end[3]);
/* propagation_and_undist's back-propagation loop (IMU_Processing.hpp:390-415). poses: the IMUpose table, npose x 22 doubles
 * {offset_time, acc[3], gyr[3], vel[3], pos[3], rot[9]} (Pose6D, common_lib.h:184-199); the state is the propagated one.
 * 2 <= npose <= LIINIT_MAX_IMU_POSES. */
#define LIINIT_MAX_IMU_POSES 4096
int liinit_raw_undistort_imu(liinit_ctx* h, const double* poses, int npose, const double rot_end[9], const double pos_end[3],
                             const double R_LI[9], const double T_LI[3]);
/* ---- cut-frame preprocess (Preprocess::process_cut_frame_livox / _pcl2, src/preprocess.cpp:50-335): one driver message ->
 * decoded, filtered, time-sorted, cut and re-timed sub-frames, kept on the device. A cut writes one of LIINIT_FRAME_SLOTS message
 * slots (round robin); each returned sub-frame carries a handle that liinit_frame_stage turns into the staged raw cloud, exactly as
 * liinit_raw_upload(pts12, 12, 9, n) of the same points would. A message that yields no sub-frame does not take a slot. The buffers
 * are allocated on the first cut. Errors: LIINIT_ERR_CAPACITY when n exceeds the raw staging capacity (max(max_scan_points, 2^20))
 * or required_cut_num exceeds cap; LIINIT_ERR_INVALID for a bad lidar_type / point_filter_num / required_frame_num / layout, or
 * (spinning sensors whose offset times come from the rotation model) a ring >= 128. Every error leaves the context as it was. */
#define LIINIT_FRAME_SLOTS 4
#define LIINIT_FRAME_MAX_CUT 256     /* largest required_frame_num */
#define LIINIT_LIDAR_AVIA 1          /* Livox CustomMsg (preprocess.h LID_TYPE) */
#define LIINIT_LIDAR_VELO 2          /* PointCloud2: velodyne_ros::Point {x,y,z,intensity f32, time f32, ring u16} */
#define LIINIT_LIDAR_OUSTER 3        /* ouster_ros::Point {.., intensity f32, t u32, ring u8} */
#define LIINIT_LIDAR_PANDAR 5        /* pandar_ros::Point {.., intensity f32, timestamp f64, ring u16} */
#define LIINIT_LIDAR_ROBOSENSE 6     /* robosense_ros::Point {.., intensity u8, ring u16, timestamp f64} */
typedef struct liinit_frame_params {
    int lidar_type;          /* preprocess/lidar_type */
    int N_SCANS;             /* preprocess/scan_line */
    double blind;            /* preprocess/blind [m] */
    int point_filter_num;    /* point_filter_num */
    int required_frame_num;  /* cut_frame_num: sub-frames per message once scan_count passes 5 (Livox) / 20 (PointCloud2) */
    int scan_count;          /* the node's scan_count for this message (incremented before the cut, laserMapping.cpp:317,355) */
    double stamp;            /* msg->header.stamp.toSec() [s] */
} liinit_frame_params;
typedef struct liinit_pcl2_layout {
    int point_step;          /* bytes per point */
    int off_x, off_y, off_z, off_intensity, off_time, off_ring;   /* byte offsets of the fields; -1 = absent (reads as 0) */
} liinit_pcl2_layout;
typedef struct liinit_subframe {
    long long handle;        /* for liinit_frame_stage / liinit_frame_download */
    double t_beg;            /* time_buffer entry: last_frame_end_time / 1000 [s] */
    float end_ms;            /* curvature of the last point [ms]; lidar_end_time = t_beg + end_ms / 1000 */
    int n;                   /* points */
} liinit_subframe;
/* pts: n Livox CustomPoint records {u32 offset_time [ns]; f32 x, y, z; u8 reflectivity, tag, line}, stride_bytes >= 19 apart
 * (19 on the wire, 20 as the ROS struct). out[0 .. *n_sub) receives the sub-frames in time order (0 or required_cut_num of them). */
int liinit_frame_cut_livox(liinit_ctx* h, const void* pts, int stride_bytes, int n, const liinit_frame_params* p, liinit_subframe* out,
                           int cap, int* n_sub);
/* data: the PointCloud2 data buffer (little endian), n = width * height points of layout->point_step bytes. */
int liinit_frame_cut_pcl2(liinit_ctx* h, const void* data, const liinit_pcl2_layout* layout, int n, const liinit_frame_params* p,
                          liinit_subframe* out, int cap, int* n_sub);
/* The sub-frame becomes the staged raw cloud (time = re-timed curvature). LIINIT_ERR_INVALID when its slot has been reused. */
int liinit_frame_stage(liinit_ctx* h, long long handle);
/* The sub-frame in the 12-float PointType layout: x, y, z, 1, normals 0, intensity, curvature, 0, 0. *n = its size; pts12 may
 * be NULL to ask for it; LIINIT_ERR_CAPACITY when cap_points < *n (nothing written). */
int liinit_frame_download(liinit_ctx* h, long long handle, float* pts12, int cap_points, int* n);
/* The staged raw cloud as packed xyz (after whatever undistortion ran). */
int liinit_raw_download(liinit_ctx* h, float* xyz, int cap_points, int* n);
/* The staged (undistorted) raw cloud in the world frame, packed xyz in upload order: pointBodyToWorld (laserMapping.cpp:209-220)
 * with the given state, the same arithmetic as the map update. This is feats_undistort as publish_frame_world publishes it with
 * dense_publish_en (:563) and as pcd_save accumulates it (:594-603); liinit_cloud_download returns it with its attributes.
 * *n = number of staged points; xyz may be NULL to ask for it. LIINIT_ERR_CAPACITY when cap_points < *n (nothing is written),
 * LIINIT_ERR_INVALID when no raw cloud is staged. */
int liinit_raw_download_world(liinit_ctx* h, const double rot_end[9], const double pos_end[3], const double R_LI[9], const double T_LI[3],
                              float* xyz, int cap_points, int* n);
/* downSizeFilterSurf.filter (laserMapping.cpp:917-918): voxel grid over the staged cloud -> the resident scan. */
int liinit_raw_downsample(liinit_ctx* h, float leaf_size, int* n_down);
/* Raw (undistorted, not yet downsampled) scan: voxel-grid filter on the device, then the result becomes the resident scan.
 * Replaces downSizeFilterSurf.setInputCloud/filter (laserMapping.cpp:122,823,917-918 = PCL VoxelGrid, leaf = mapping/filter_size_surf)
 * followed by liinit_scan_upload. n_down = feats_down_size. Output order: ascending leaf index, as PCL. */
int liinit_scan_upload_raw(liinit_ctx* h, const float* xyz, int stride_floats, int n, float leaf_size, int* n_down);
/* The resident scan (feats_down_body) as packed xyz. */
int liinit_scan_download_body(liinit_ctx* h, float* xyz, int cap_points, int* n);
/* One ICP pass, laserMapping.cpp:959-1071 + the reduction of :1080.
 *   rot_end, pos_end, R_LI (offset_R_L_I), T_LI (offset_T_L_I): the pose part of StatesGroup (common_lib.h:160-163).
 *   imu_en: 12-column Jacobian (:1054-1062) else 6 columns (:1063-1066).
 *   nearest_search_en: search pass (:978-985) or reuse of stored neighbours and flags (:989-994).
 * Outputs (host): HtH[144] = Hsub^T Hsub (UNWEIGHTED; the reference's R_inv=1000 (:1050) is applied by the
 * caller), Htr[12] = Hsub^T meas_vec with meas = -pd2 (:1070), m = effect_feat_num (:1012-1020).
 * res_sq (optional, may be NULL) = sum of pd2^2 over the selected points. */
int liinit_icp_iterate(liinit_ctx* h, const double rot_end[9], const double pos_end[3], const double R_LI[9],
                       const double T_LI[3], int imu_en, int nearest_search_en, double HtH[144], double Htr[12], int* m,
                       double* res_sq);
/* Same pass, results left on the device: d_out = device pointer to 160 doubles
 * [HtH 144 | Htr 12 | res_sq | m | pad 2], written on the context's stream; no host synchronisation.
 * With a communicator attached (liinit_comm_init) both forms return the SUM over the ranks. */
int liinit_icp_iterate_device(liinit_ctx* h, const double rot_end[9], const double pos_end[3], const double R_LI[9],
                              const double T_LI[3], int imu_en, int nearest_search_en, double* d_out160);
/* laserCloudOri / corr_normvect after compaction (laserMapping.cpp:1013-1020; published at :625-636):
 * ori_xyz [cap*3] body points, normvec [cap*4] = (nx,ny,nz,pd2), order preserved. */
int liinit_scan_download_effect(liinit_ctx* h, float* ori_xyz, float* normvec, int cap_points, int* m);
/* Per-point state of the last pass for parity tests (any pointer may be NULL): world [n*3] (feats_down_world),
 * near_xyz [n*5*3] + near_cnt [n] (Nearest_Points), selected [n] (point_selected_surf), normvec [n*4]. */
int liinit_scan_download_state(liinit_ctx* h, float* world_xyz, float* near_xyz, int* near_cnt, unsigned char* selected,
                               float* normvec);
/* ---- published clouds (publish_frame_world, publish_frame_body, publish_effect_world and pcd_save, laserMapping.cpp:561-636) ----
 * One cloud as 48-byte pcl::PointXYZINormal records, 12 floats {x, y, z, 1, normal_x, normal_y, normal_z, 0, intensity, curvature, 0, 0}:
 * the data of the sensor_msgs/PointCloud2 that pcl::toROSMsg makes of a PointCloudXYZI (point_step 48; FLOAT32 fields x@0, y@4, z@8,
 * normal_x@16, normal_y@20, normal_z@24, intensity@32, curvature@36; the padding floats are 0). The world-frame clouds are
 * pointBodyToWorld (:209-220) with the given state into fresh points: xyz transformed, normals and intensity copied, curvature 0.
 *   REGISTERED       the staged, undistorted raw cloud (feats_undistort) in staging order; xyz bit-equal to liinit_raw_download_world.
 *                    Normals and intensity: floats 4-6 and 8 of a liinit_raw_upload(pts, >= 12, 9, n) point, the message intensity of a
 *                    liinit_frame_stage sub-frame (normals 0), zeros for any other upload.
 *   REGISTERED_DOWN  the resident scan (feats_down_body) made by liinit_raw_downsample: normals and intensity are leaf means, as PCL's
 *                    VoxelGrid with downsample_all_data_ computes them (input-order sums, divided by the count like the xyz); zeros
 *                    for a scan uploaded as xyz.
 *   BODY             the staged, undistorted raw cloud as it is: curvature = its time offset [ms]. The pose arguments may be NULL.
 *   EFFECT           laserCloudOri: the resident-scan points the last ICP pass selected, in index order (effect_feat_num of them, the
 *                    count liinit_scan_download_effect returns), intensity sqrt(1000) as the Jacobian loop leaves it (:1050-1051).
 *                    With a communicator attached this is collective (the flags of every rank's slot are all-gathered first); every rank
 *                    receives the whole frame's cloud.
 * rec12 may be NULL to ask for *n. LIINIT_ERR_CAPACITY when cap_points < *n (nothing written). LIINIT_ERR_INVALID for an unknown
 * `which`, no staged raw cloud (REGISTERED, BODY), no resident scan (REGISTERED_DOWN), no ICP pass on the resident scan (EFFECT).
 * No call changes any state: the update and map_incremental give the same results with or without these calls in between. */
#define LIINIT_CLOUD_REGISTERED 1       /* feats_undistort -> world  (publish_frame_world with dense_pub_en; pcd_save) */
#define LIINIT_CLOUD_REGISTERED_DOWN 2  /* feats_down_body -> world  (publish_frame_world without dense_pub_en) */
#define LIINIT_CLOUD_BODY 3             /* feats_undistort as it is  (publish_frame_body) */
#define LIINIT_CLOUD_EFFECT 4           /* laserCloudOri -> world    (publish_effect_world) */
int liinit_cloud_download(liinit_ctx* h, int which, const double rot_end[9], const double pos_end[3], const double R_LI[9],
                          const double T_LI[3], float* rec12, int cap_points, int* n);
/* map_incremental (laserMapping.cpp:516-559) with the final state; uses the neighbour lists retained on the
 * device by the last search pass. ds = the node's double filter_size_map_min. n_add / n_no_downsample:
 * sizes of PointToAdd / PointNoNeedDownsample. */
int liinit_map_incremental(liinit_ctx* h, const double rot_end[9], const double pos_end[3], const double R_LI[9],
                           const double T_LI[3], double ds, int flg_EKF_inited, int* n_add, int* n_no_downsample);

/* ---- device-pointer twins: clouds that are already on the GPU (a PyTorch pipeline, a simulator) ----------------------------------
 * Each function behaves like its host twin named in its comment -- same arguments, layouts, error codes and results, bit for bit --
 * except that its point arrays are memory of the context's device instead of host memory.
 *   Pointers: every point array (input or output) must be cudaMemoryTypeDevice or cudaMemoryTypeManaged memory of the context's
 *     device (cudaPointerGetAttributes). Otherwise, and for a null array where the twin needs one, the call returns LIINIT_ERR_INVALID,
 *     liinit_last_error names the argument, and NOTHING changes: map, resident scan, staged cloud and liinit_launch_count are as before.
 *     A stride-4 input that is 16-byte aligned is read as float4 in place; any other input is repacked from the caller's memory.
 *   Stream order: the work is queued on the context's stream (liinit_set_stream / liinit_get_stream). An input only has to be ready on
 *     that stream when the call is made, an output is valid once that stream reaches it, and an input may be reused once that stream
 *     has passed the call. A call synchronises only where its twin returns a host scalar that the device computes: the map updates
 *     (capacity errors, `added`), the host count of an EFFECT cloud, and the brick count that sizes a map download.
 *   With a communicator attached (liinit_comm_init) every device twin returns LIINIT_ERR_INVALID: the device frame is not cut into
 *   rank slots. */
/* The stream the context runs on (its own, or the one given to liinit_set_stream), as a cudaStream_t. */
int liinit_get_stream(liinit_ctx* h, void** cuda_stream);
/* liinit_map_build: xyz read in place (stride 4, aligned) or repacked on the device. Synchronises once at the end (capacity errors). */
int liinit_map_build_device(liinit_ctx* h, const float* xyz, int stride_floats, int n);
/* liinit_map_add_points: *added returned to the host as the twin does (one synchronisation per 2^20-point chunk). */
int liinit_map_add_points_device(liinit_ctx* h, const float* xyz, int stride_floats, int n, int downsample_on, int* added);
/* liinit_scan_upload: stride 4 is one device-to-device copy, 3 and 12 are repacked from the caller's memory. No synchronisation. */
int liinit_scan_upload_device(liinit_ctx* h, const float* body_xyz, int stride_floats, int n);
/* liinit_raw_upload: repacked from the caller's memory; the PointType layout (stride >= 12, time_index 9) brings normals and intensity
 * along as the twin does. No synchronisation. */
int liinit_raw_upload_device(liinit_ctx* h, const float* pts, int stride_floats, int time_index, int n);
/* liinit_map_nearest_search: queries, out_xyz [n*5*3], out_d2 [n*5] and out_cnt [n] on the device (any output may be NULL). Both
 * twins run the same kernels, count and PointType_CMP tie order (ikd_Tree.h:57-60, applied when both out_xyz and out_d2 are given)
 * included; the host twin only adds the copies of the queries and the results. No synchronisation, any n. */
int liinit_map_nearest_search_device(liinit_ctx* h, const float* q_xyz, int stride_floats, int n, double max_dist, float* out_xyz,
                                     float* out_d2, int* out_cnt);
/* liinit_cloud_download: the records are built in rec12 itself, which must be 16-byte aligned. n (host, may be NULL) and d_n (device,
 * may be NULL) receive the point count. REGISTERED, BODY and REGISTERED_DOWN never synchronise. EFFECT synchronises only when n is
 * given or when cap_points is smaller than the resident scan (the count must then be known before anything is written). */
int liinit_cloud_download_device(liinit_ctx* h, int which, const double rot_end[9], const double pos_end[3], const double R_LI[9],
                                 const double T_LI[3], float* rec12, int cap_points, int* n, int* d_n);
/* liinit_map_download: the live points as packed xyz into xyz [cap_points*3], their number into *d_n (device, required; counts past
 * cap_points are not written, as in the twin). Synchronises once for the brick count that sizes the launch. */
int liinit_map_download_device(liinit_ctx* h, float* xyz, int cap_points, int* d_n);

/* Test hook: esti_plane<double>(pabcd, points, 0.1) (include/common_lib.h:236-269) of the device for n independent neighbour sets.
 * nb_xyz [n*15] = five xyz per set (f32), pabcd [n*4] = (nx, ny, nz, d), valid [n]. The very function the plane pass calls. */
int liinit_debug_esti_plane(liinit_ctx* h, const float* nb_xyz, int n, double* pabcd, unsigned char* valid);

/* multi-GPU (SURVEY.md section 8e; the reference is single-process, its only parallelism the OpenMP loop laserMapping.cpp:964-968) --------
 * One process (or thread) per GPU, one context each. The map is REPLICATED: every rank makes the same map calls with the same data.
 * The scan is SHARDED: every rank uploads the same whole frame, the library cuts it into nranks equal slots and the search / plane
 * kernels of a rank work on its slot only. The one exchange of the path -- the sum of [HtH 144 | Htr 12 | res_sq | m] over the ranks
 * (one ncclAllReduce of 160 doubles over NVLink on the context's stream) -- happens INSIDE liinit_icp_iterate / _device, so the
 * host-side IESKF loop (liinit_scan_update, liinit_host.h) is unchanged and every rank ends a scan with the same state.
 * liinit_map_incremental and the download hooks first all-gather the per-point results (Nearest_Points copies, flags, normals) of the
 * other ranks' slots, then every rank applies the whole frame's update to its replica: collective calls, same order on every rank.
 * NCCL is loaded with dlopen("libnccl.so.2") when the first of these functions is called; single-GPU use never touches it.
 * How the sum travels: with one process per GPU on an NVLink node, liinit_comm_init maps every rank's 2.6 kB exchange buffer into every
 * process (CUDA IPC) and the LAST BLOCK of the plane kernel does the collective itself -- peer stores of its 160 doubles into every rank's
 * buffer, a system-scope flag, a spin on the other ranks' flags, a rank-ordered sum (bit-identical on every rank): no extra launch, no
 * NCCL kernel. If any rank cannot map its peers (ranks as threads of one process, no peer access) or LIINIT_COMM_MODE=nccl is set, all
 * ranks use ncclAllReduce on the context's stream instead. NCCL always carries the set-up and the all-gathers of per-point results.
 * As with any collective: a rank that does not make the call (it returned an error earlier, or died) leaves the others waiting -- the
 * spin in the plane kernel has no time-out, exactly like a pending ncclAllReduce; supervise the ranks from outside. */
#define LIINIT_COMM_ID_BYTES 128
/* ncclGetUniqueId: call on ONE rank, hand the 128 bytes to the others through whatever channel the application has. */
int liinit_comm_unique_id(void* id128);
/* ncclCommInitRank on the context's device; collective over the nranks contexts. LIINIT_ERR_CUDA if NCCL is missing. */
int liinit_comm_init(liinit_ctx* h, const void* id128, int nranks, int rank);
/* This rank's OWN accumulator block of the last pass (before the sum), 160 doubles to the host: lets an application / the bench
 * verify the reduction (sum of the ranks' blocks == what liinit_icp_iterate returned). */
int liinit_comm_last_local(liinit_ctx* h, double* out160);
/* 1 if the accumulators are summed over peer memory inside the plane kernel, 0 if by ncclAllReduce (or no communicator). */
int liinit_comm_mode(liinit_ctx* h, int* peer_memory);
/* nranks / rank of the context and the slot [shard_lo, shard_lo + shard_n) of the resident frame this rank works on. */
int liinit_comm_info(liinit_ctx* h, int* nranks, int* rank, int* shard_lo, int* shard_n);

/* A scan is searched more than once (laserMapping.cpp:1102-1106: rematch after convergence / at the last but one iteration). By default
 * the later search passes of a scan are SEEDED: the five neighbours the previous pass stored still exist in the map (the library tracks
 * every call that can remove a point), so their largest distance from the moved query bounds the new 5th-neighbour distance -- one shell,
 * hardly any inserts, same result bit for bit. enabled = 0 makes every search pass start from scratch (what bench.py times as the metric:
 * the FIRST search pass of a scan). */
int liinit_set_reseed(liinit_ctx* h, int enabled);

/* instrumentation (the reference has none around this loop, SURVEY.md section 5) ---- */
/* Device time in milliseconds of the kernels of the last liinit_icp_iterate* call (CUDA events on the context's
 * stream) and the number of kernel launches it made. */
int liinit_last_pass_timing(liinit_ctx* h, float* kernel_ms, int* launches);
/* Per-kernel device times of the last pass: the 5-NN kernel (0 for a reuse pass) and the plane/Jacobian/reduction kernel. */
int liinit_last_pass_kernel_times(liinit_ctx* h, float* knn_ms, float* plane_ms);
/* The spatial index this context searches (LIINIT_KNN_BRICKS / LIINIT_KNN_CELLS) after defaults were resolved. */
int liinit_knn_index(liinit_ctx* h, int* knn_index);
/* Cumulative number of kernels launched by this context. */
int liinit_launch_count(liinit_ctx* h, long long* launches);
/* Map statistics: bricks in use, hash slots, pool points in use / capacity. */
int liinit_map_stats(liinit_ctx* h, int* bricks, int* hash_slots, long long* pool_used, long long* pool_cap);

/* map assessment (DESIGN.md section 4d) ----------------------------------------------------------------------------------------------
 * Scores an extrinsic by how sharp a map it builds. The store holds staged (undistorted, body-frame) clouds with the pose and extrinsic
 * of their update. An evaluation places every stored point with li_body_to_world (fp64, f32 store) using its scan's rot_end / pos_end
 * and either the scan's own extrinsic (as_run) or a candidate (R_LI, T_LI). Every s-th stored point is a query. Its neighbourhood is
 * every stored point with d2 <= r2, d2 = ((dx*dx + dy*dy) + dz*dz) of the fp64 offsets; the query itself is included. The fp64 moments
 * of the offsets give Sigma = S2/n - m m^T. With n >= min_neighbors and det Sigma > 0 the query is valid:
 * h = 1/2 (3 ln(2 pi e) + ln det Sigma), v = lambda_min(Sigma). Otherwise it is sparse (n < min_neighbors) or degenerate (det <= 0).
 * MME = mean h and MPV = mean v over the valid queries. Moments are summed in a fixed candidate order and the totals in query order,
 * so an evaluation is bit-identical from call to call and independent of the launch shape and the SM count.
 * Every call returns LIINIT_ERR_INVALID, and changes nothing, before liinit_assess_reserve and under a communicator. */
#define LIINIT_ASSESS_MAX_QUERIES 2000000    /* queries per evaluation; the automatic stride is the smallest that stays within it */
#define LIINIT_ASSESS_MAX_POINTS (1ll << 30)
#define LIINIT_ASSESS_MAX_SCANS (1 << 24)
typedef struct {
    double radius;        /* r [m], > 0 and finite */
    int min_neighbors;    /* n_min, >= 4 */
    int query_stride;     /* s; 0 = automatic */
    int as_run;           /* 1: every scan with its own stored extrinsic; R_LI / T_LI may then be NULL */
    int reserved;
} liinit_assess_params;
typedef struct {
    long long points;     /* stored points placed */
    long long queries;
    int stride;           /* s used */
    int scans;            /* stored scans */
    long long valid, sparse, degenerate;
    double mme, mpv;      /* NaN when no query is valid */
} liinit_assess_result;
/* Allocates the store (max_points points, max_scans scans) and the evaluation buffers, about 110 bytes per point. Calling it again
 * clears the store. LIINIT_ERR_INVALID for max_points outside [1, LIINIT_ASSESS_MAX_POINTS] or max_scans outside
 * [1, LIINIT_ASSESS_MAX_SCANS]. */
int liinit_assess_reserve(liinit_ctx* h, long long max_points, int max_scans);
/* Appends the staged cloud (the BODY cloud of liinit_cloud_download) with its update's pose and extrinsic: a device-to-device copy, no
 * synchronisation. When the store has no room for it, nothing is stored, the scan is counted as skipped and *appended = 0
 * (LIINIT_OK). LIINIT_ERR_INVALID when no raw cloud is staged. */
int liinit_assess_append(liinit_ctx* h, const double rot_end[9], const double pos_end[3], const double R_LI[9], const double T_LI[3],
                         int* appended);
/* Stored points and scans, and scans skipped for lack of room (any pointer may be NULL). */
int liinit_assess_info(liinit_ctx* h, long long* points, int* scans, int* skipped);
/* One evaluation (synchronises). Leaves the map, the staged cloud, the resident scan and the ICP state untouched.
 * LIINIT_ERR_INVALID: radius <= 0 or not finite, min_neighbors < 4, query_stride < 0, an empty store, a non-finite or missing
 * candidate. LIINIT_ERR_CAPACITY: more than LIINIT_ASSESS_MAX_QUERIES queries for the given stride, or a placed point that is not
 * finite, lies 2^30 cells or more from the origin, or makes the cloud span more cells than a 63-bit key holds. */
int liinit_assess_evaluate(liinit_ctx* h, const liinit_assess_params* p, const double R_LI[9], const double T_LI[3], liinit_assess_result* out);
/* Per-query values of the last evaluation, in query order (query j is stored point j * stride): h, v (NaN for a sparse or degenerate
 * query) and the neighbour count. *n = queries; any output may be NULL; LIINIT_ERR_CAPACITY when cap < queries. */
int liinit_assess_download(liinit_ctx* h, double* h_out, double* v_out, int* n_out, long long cap, long long* n);
/* Test hook: the points the last evaluation placed, xyz [cap*3] in stored order. *n = their number; xyz may be NULL. After a
 * liinit_assess_cloud they are the points that call placed. */
int liinit_assess_download_placed(liinit_ctx* h, float* xyz, long long cap, long long* n);
/* Where the map is blurred: every stored point is a query (p->query_stride must be 0 or 1), placed and cell-sorted once, its moments
 * summed in batches of at most LIINIT_ASSESS_MAX_QUERIES stored points. Point i's h, v and neighbour count are bit-equal to query i / s
 * of a liinit_assess_evaluate with stride s dividing i and the same extrinsic. Records are 8 floats,
 * x y z entropy plane_variance neighbors points valid:
 *   leaf == 0: one per stored point, in stored order: the placed point, (float) h, v and n, points = 1, valid = 1 or 0 (h, v NaN).
 *   leaf > 0:  one per occupied cubic leaf of edge leaf (leaf = floor(w / leaf) per axis, keyed over the placed bounding box like the
 *              cells), in ascending key. fp64 sums of the leaf's per-point records, in stored order, stored as float: the centroid
 *              and the mean neighbour count over all its points, mean h and v over its valid points (NaN when none is valid), the
 *              point count and the valid count.
 * rec8 == NULL asks for the number of records, *n (with totals == NULL too, nothing but the count is computed). *n is always set;
 * cap_records < *n returns LIINIT_ERR_CAPACITY and writes neither rec8 nor totals. totals (may be NULL): the full-resolution counts,
 * MME and MPV over every stored point (queries = points, stride 1). Records reach the host in chunks through the staging buffer;
 * synchronises. Leaves the map, the staged cloud, the resident scan, the ICP state and the last evaluation's per-query values
 * (liinit_assess_download) untouched. Errors as liinit_assess_evaluate, and LIINIT_ERR_INVALID for query_stride other than 0 or 1 or a
 * negative or non-finite leaf; LIINIT_ERR_CAPACITY for a leaf so small that a placed point lies 2^30 leaves or more from the origin
 * or the cloud spans more leaves than a 63-bit key holds. No device memory beyond liinit_assess_reserve's. */
int liinit_assess_cloud(liinit_ctx* h, const liinit_assess_params* p, const double R_LI[9], const double T_LI[3], double leaf, float* rec8,
                        long long cap_records, long long* n, liinit_assess_result* totals);

/* The timed store (DESIGN.md section 4d): it also keeps what the IMU undistortion of a scan needs, so an evaluation can redo it for a
 * candidate extrinsic and a candidate time lag. A timed scan is one whose staged cloud was held (liinit_assess_hold) before
 * liinit_raw_undistort_imu and appended with liinit_assess_append_timed: its raw points (xyz, time [ms]), its pose table and the
 * propagated state of that call. Every other stored scan is untimed and is placed from its stored points at every lag. The stored
 * points, their order and everything liinit_assess_evaluate / _cloud / _download return are those of the plain store. */
#define LIINIT_ASSESS_MAX_POSE_ROWS (1ll << 30)
typedef struct {
    const double* poses;  /* npose x 22 doubles (Pose6D), host memory, as passed to liinit_raw_undistort_imu */
    int npose;            /* 2 <= npose <= LIINIT_MAX_IMU_POSES */
    int reserved;
    double rot[9], pos[3];    /* the propagated state passed to liinit_raw_undistort_imu: rot_end, pos_end ... */
    double R_LI[9], T_LI[3];  /* ... and its extrinsic */
    double vel[3];            /* the propagated vel_end */
} liinit_assess_timing;
/* liinit_assess_reserve, plus a raw-point buffer (16 bytes per point), a timing record per scan (about 400 bytes) and a pool of
 * max_pose_rows pose rows (176 bytes each). Calling it (or liinit_assess_reserve) again clears the store. LIINIT_ERR_INVALID also for
 * max_pose_rows outside [2, LIINIT_ASSESS_MAX_POSE_ROWS]. */
int liinit_assess_reserve_timed(liinit_ctx* h, long long max_points, int max_scans, long long max_pose_rows);
/* Holds the staged raw cloud for the next liinit_assess_append_timed: a device-to-device copy behind the stored points, no
 * synchronisation. Call it between staging the cloud and liinit_raw_undistort_imu. Any later staging call (raw upload, frame stage,
 * a map or scan upload) or append ends the hold. LIINIT_ERR_INVALID when no raw cloud is staged or the store is not timed. */
int liinit_assess_hold(liinit_ctx* h);
/* liinit_assess_append (the staged, undistorted cloud with the posterior pose and extrinsic), and commits the held raw points, the
 * pose table and the prior state *t. No room for the points or the scan: skipped as by liinit_assess_append. No room in the pose pool:
 * stored as an untimed scan. LIINIT_ERR_INVALID when the store is not timed, no hold of the current staged cloud exists, the held and
 * staged clouds differ in size, or t->npose is outside [2, LIINIT_MAX_IMU_POSES]. In a timed store, liinit_assess_append stores an
 * untimed scan. */
int liinit_assess_append_timed(liinit_ctx* h, const double rot_end[9], const double pos_end[3], const double R_LI[9], const double T_LI[3],
                               const liinit_assess_timing* t, int* appended);
/* Timed and untimed stored scans and pose rows in use (any pointer may be NULL). LIINIT_ERR_INVALID for a store that is not timed. */
int liinit_assess_timing_info(liinit_ctx* h, int* timed_scans, int* untimed_scans, long long* pose_rows);
/* liinit_assess_evaluate with every timed scan re-undistorted for the candidate extrinsic (as_run: the prior extrinsic for the
 * undistortion, each scan's posterior one for the placement) and the lag shift [s]: the candidate's total lag is the run's + lag_shift,
 * so a point at tau [ms] is undistorted at t = tau / 1000 + lag_shift in the run's table, head row as liinit_raw_undistort_imu's
 * (none: untouched at lag_shift 0, row 0 otherwise), towards rot_end Exp(gyr_last, lag_shift) and pos_end + vel_end lag_shift +
 * 1/2 acc_last lag_shift^2 (the table's last row). At lag_shift 0 as-run it is bit-equal to liinit_assess_evaluate as-run.
 * liinit_assess_download / _download_placed then return this evaluation's values. Errors as liinit_assess_evaluate, and
 * LIINIT_ERR_INVALID for a store that is not timed or a non-finite lag_shift. */
int liinit_assess_evaluate_timed(liinit_ctx* h, const liinit_assess_params* p, const double R_LI[9], const double T_LI[3], double lag_shift,
                                 liinit_assess_result* out);
/* Empties the store (plain or timed) and keeps its reservation: no stored point, scan, skip, pose row or evaluation. */
int liinit_assess_clear(liinit_ctx* h);

/* LIO-phase replay (DESIGN.md section 4d): run the LIO loop again from the hand-over for a candidate calibration ------------------------
 * liinit_map_snapshot copies the whole map state device to device on the context's stream: hash table, the used part of the brick list
 * and of the point pool, the counters, the cell directory when there is one, and the staged raw cloud (the cloud the scan after the
 * hand-over downsamples again). liinit_map_restore copies it back: every map entry point then behaves as it did at the snapshot, and the
 * staged raw cloud is the snapshot's. The first snapshot allocates the hash-sized buffers; the pool and staging copies grow on demand.
 * *bytes (may be NULL): bytes the snapshot copied. liinit_map_restore without a snapshot: LIINIT_ERR_INVALID. */
int liinit_map_snapshot(liinit_ctx* h, long long* bytes);
int liinit_map_restore(liinit_ctx* h);
/* The replay store keeps sub-frames as liinit_frame_stage would stage them: xyz and time [ms] (16 bytes per point), intensity (4 bytes)
 * and each sub-frame's lidar_beg_time and end offset [ms]. liinit_replay_reserve allocates it (again: clears it). */
int liinit_replay_reserve(liinit_ctx* h, long long max_points, int max_frames);
/* Copies sub-frame `handle` (liinit_frame_cut_*) into the store, device to device, with its t_beg [s] and end_ms. A sub-frame that does
 * not fit is skipped and counted (*appended = 0). LIINIT_ERR_INVALID without a reserve or for an unknown handle. */
int liinit_replay_append(liinit_ctx* h, long long handle, double t_beg, float end_ms, int* appended);
/* Stored sub-frames, skipped ones and stored points (any pointer may be NULL). */
int liinit_replay_info(liinit_ctx* h, int* frames, int* skipped, long long* points);
/* t_beg, end_ms and point count of stored sub-frame j (any pointer may be NULL). */
int liinit_replay_frame(liinit_ctx* h, int j, double* t_beg, float* end_ms, int* n);
/* Stages stored sub-frame j as the raw cloud, exactly as liinit_frame_stage staged the original. */
int liinit_replay_stage(liinit_ctx* h, int j);
/* Concurrent replays: one context per replay, all reading one store. After liinit_replay_share(worker, lead), the worker's
 * liinit_map_restore copies from the lead's snapshot and its liinit_replay_info / _frame / _stage read the lead's store. The pointers
 * are not owned: the worker allocates no copy of either. The call synchronises the lead's stream once, so the store and the snapshot
 * are complete before any worker's stream reads them; each context then runs on its own stream, and a worker and its lead (or two
 * workers) may be driven from distinct threads at once. The worker keeps its own map, staged cloud, resident scan and assessment store.
 * LIINIT_ERR_INVALID, with a message, when: worker == lead; they are on different devices; their configurations differ (hash slots,
 * brick cells, cell directory on or off, capacities, filter_size_map); either has a communicator; the worker already shares or is
 * itself a lead; the lead shares another's; the lead has no snapshot or no replay store.
 * While shared: on the lead, liinit_map_snapshot, liinit_replay_reserve, liinit_replay_append and liinit_destroy are refused; on the
 * worker, liinit_map_snapshot, liinit_replay_reserve and liinit_replay_append are refused (LIINIT_ERR_INVALID).
 * liinit_replay_unshare (LIINIT_ERR_INVALID when the context does not share) and liinit_destroy of the worker end the sharing; both
 * first synchronise the worker's stream. */
int liinit_replay_share(liinit_ctx* worker, liinit_ctx* lead);
int liinit_replay_unshare(liinit_ctx* worker);

#ifdef __cplusplus
}
#endif
#endif /* LIINIT_GPU_H */
