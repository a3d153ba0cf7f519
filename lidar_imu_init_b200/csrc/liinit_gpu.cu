// liinit_gpu.cu -- C-ABI implementation (include/liinit_gpu.h) over the sm_90a kernels.
//
// One context = one GPU, one stream, one device-resident map, one resident scan. No CPU fallback:
// every entry point fails with LIINIT_ERR_CUDA if the CUDA runtime reports an error.
#include "../../include/liinit_gpu.h"

#include <cuda_runtime.h>
#ifdef LI_SIMT_EMUL
#include "device_memory_emul.h"   // CPU checker only (tests/emul): tells its cudaMalloc memory from host memory
#endif
#ifndef LI_SIMT_EMUL
#include <dlfcn.h>
#include <nccl.h>   // types only: the library is dlopen()ed when a communicator is asked for (no link-time dependency)
#endif

#include <atomic>
#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "common.cuh"
#include "icp_kernels.cuh"
#include "knn_kernels.cuh"
#include "cells.cuh"
#include "map_kernels.cuh"
#include "voxelgrid_kernels.cuh"
#include "undistort_kernels.cuh"
#include "preprocess_kernels.cuh"
#include "output_kernels.cuh"
#include "assess_kernels.cuh"
#include "assess_time_kernels.cuh"

#ifndef LI_CELLS_MINB
#define LI_CELLS_MINB 6
#endif
#ifndef LIINIT_KNN_DEFAULT
#define LIINIT_KNN_DEFAULT LIINIT_KNN_BRICKS   // what knn_index = 0 selects
#endif


namespace {

thread_local std::string g_create_error;

#ifndef LI_SIMT_EMUL
// NCCL entry points, resolved at run time from libnccl.so.2 (the copy the process already has -- e.g. the one a PyTorch host
// application loaded -- or the system one). A single-GPU deployment never touches it.
struct NcclApi {
    void* lib = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    std::string err;
};
NcclApi* nccl_api() {
    static NcclApi api;
    static bool tried = false;
    if (tried) return api.lib ? &api : nullptr;
    tried = true;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* nm : names) {
        api.lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
        if (api.lib) break;
    }
    if (!api.lib) {
        api.err = std::string("dlopen(libnccl.so.2): ") + dlerror();
        return nullptr;
    }
    bool ok = true;
    auto sym = [&](const char* n) { void* f = dlsym(api.lib, n); if (!f) { ok = false; api.err = std::string("missing NCCL symbol ") + n; } return f; };
    api.GetUniqueId = (decltype(api.GetUniqueId))sym("ncclGetUniqueId");
    api.CommInitRank = (decltype(api.CommInitRank))sym("ncclCommInitRank");
    api.CommDestroy = (decltype(api.CommDestroy))sym("ncclCommDestroy");
    api.AllReduce = (decltype(api.AllReduce))sym("ncclAllReduce");
    api.AllGather = (decltype(api.AllGather))sym("ncclAllGather");
    api.GetErrorString = (decltype(api.GetErrorString))sym("ncclGetErrorString");
    if (!ok) {
        dlclose(api.lib);
        api.lib = nullptr;
        return nullptr;
    }
    return &api;
}
#endif

struct Ctx {
    liinit_config cfg;
    int device = 0;
    int num_sms = 132;
    cudaStream_t own_stream = nullptr;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, evm = nullptr;
    bool last_was_search = false;
    std::string err;

    // map
    MapDev M{};
    unsigned hash_slots = 0;
    int* d_counters = nullptr;
    int* h_counters = nullptr;   // pinned
    unsigned long long* h_pool_top = nullptr;   // pinned: the bump allocator's value after the last map update
    // staging
    float* d_stage_raw = nullptr;   // strided host layout
    size_t stage_raw_floats = 0;
    float4* d_stage_pts = nullptr;  // repacked batch
    float4* d_stage_attr = nullptr; // attribute channel of the staged raw cloud: {normal_x, normal_y, normal_z, intensity} per point
    bool stage_attr = false;        // ... filled by the last raw upload / frame stage (otherwise it reads as zeros)
    int stage_pts_cap = 0;
    int* d_slot_of = nullptr;
    int* d_vslot_of = nullptr;
    int* d_flag = nullptr;
    int* d_ins = nullptr;
    int* d_vg_imin = nullptr;      // voxel-grid: first point index per leaf
    int* d_vg_block = nullptr;     // per-block counts of the effect-cloud compaction (liinit_cloud_download)
    unsigned* d_rs_keys = nullptr;  // radix sort ping-pong buffers + histogram
    unsigned* d_rs_vals = nullptr;
    int* d_rs_hist = nullptr;
    int* d_vg_misc = nullptr;      // [0..5] min/max (ordered ints), [6] out count, [7] error bits
    VgParams* d_vg_params = nullptr;
    int raw_n = 0;                          // raw (not yet downsampled) cloud staged in d_stage_pts, w = time [ms]
    long long stage_seq = 0;                // bumped by every staging call (a hold, liinit_assess_hold, is of one staged cloud)
    unsigned long long* d_tmin_idx = nullptr;
    double* d_poses = nullptr;              // IMU pose table for the undistortion (<= LIINIT_MAX_IMU_POSES x 22 doubles)
    VoxTmp V{};
    // cut-frame preprocess (liinit_frame_*), allocated on the first cut
    bool fr_ready = false;
    unsigned char* d_fr_in = nullptr;   // the message as received
    size_t fr_in_bytes = 0;
    float4* d_fr_dec = nullptr;         // decoded points by raw index: x, y, z, time [ms]
    float* d_fr_inten = nullptr;
    int* d_fr_flag = nullptr;
    unsigned* d_fr_keys = nullptr;      // (sort key, raw index) pairs; d_rs_keys / d_rs_vals are the other half of the ping-pong
    unsigned* d_fr_vals = nullptr;
    unsigned* d_fr_aux = nullptr;       // rotation model: ring by raw index, then base time by ring-sorted position
    double* d_fr_yaw = nullptr;         // rotation model: yaw [deg] by ring-sorted position
    int* d_fr_tsum = nullptr;           // two arrays of per-block counts
    int* d_fr_ring = nullptr;           // rotation model: [256] first position per ring, [256] first descent, [1] survivors
    FrameTable* d_fr_tab = nullptr;
    FrameTable* h_fr_tab = nullptr;     // pinned
    float4* d_fr_slot_pts = nullptr;    // LIINIT_FRAME_SLOTS x stage_pts_cap re-timed, sorted points (sorted index j at j - 1)
    float* d_fr_slot_inten = nullptr;
    long long fr_seq = 0;               // cuts that produced sub-frames; message fr_seq goes to slot fr_seq % LIINIT_FRAME_SLOTS
    long long fr_slot_seq[LIINIT_FRAME_SLOTS] = {};   // message held by each slot (-1: none; set when the buffers are allocated)
    int fr_slot_nsub[LIINIT_FRAME_SLOTS] = {};
    FrameSub fr_slot_sub[LIINIT_FRAME_SLOTS][LIINIT_FRAME_MAX_CUT];
    // scan
    ScanDev S{};
    float4* d_body = nullptr;
    float4* d_body_attr = nullptr;  // leaf means of the staged attribute channel for a resident scan made by liinit_raw_downsample ...
    bool body_attr = false;         // ... (an uploaded, xyz-only scan has none: zeros)
    float4* d_world = nullptr;
    int* d_near_ids = nullptr;
    float4* d_near_xyz = nullptr;
    unsigned char* d_selected = nullptr;
    float4* d_normvec = nullptr;
    int scan_n = 0;                // points of the resident scan (the whole frame)
    // multi-GPU (SURVEY.md section 8e): the map is replicated, every rank holds the whole frame and PROCESSES the shard
    // [shard_lo, shard_lo + S.n) of it; one all-reduce of the 160-double block per pass, inside liinit_icp_iterate*
    int nranks = 1, rank = 0;
    int shard_lo = 0;
#ifndef LI_SIMT_EMUL
    ncclComm_t comm = nullptr;
#endif
    double* d_acc = nullptr;       // the rank's own accumulator block (N > 1) ...
    double* d_red = nullptr;       // ... and its sum over the ranks (NCCL mode)
    // peer-memory mode (default when CUDA IPC between the ranks works): the sum happens in the last block of the plane kernel
    bool comm_p2p = false;
    void* d_xbuf = nullptr;        // this rank's exchange buffer: [2][nranks][160] doubles + [2][nranks] flags
    XchgTable* d_xtab = nullptr;   // every rank's buffer as mapped into this process
    void* peer_map[LI_MAX_RANKS] = {nullptr};   // what cudaIpcOpenMemHandle returned (closed in liinit_destroy)
    unsigned xseq = 0;             // pass sequence number (identical on every rank: the passes are collective)
    bool state_gathered = true;    // per-point results of the other ranks' shards are present on this device
    unsigned map_epoch = 0;        // bumped by everything that can REMOVE a map point (Build, downsample inserts, box delete, compaction)
    unsigned nbr_epoch = 0;        // map_epoch when the resident scan's Nearest_Points were found
    bool reseed = true;            // later search passes of a scan start from the previous pass's neighbours (liinit_set_reseed)
    bool have_neighbors = false;   // a search pass has filled near_xyz for the resident scan (point copies: map updates do not invalidate them)
    bool scan_fresh = false;   // new scan whose flags / neighbour lists have not been initialised yet (see init_scan_state)
    const float* attached = nullptr;   // device alias of a page-locked host scan not copied yet (liinit_scan_attach_host)
    int attached_stride = 0;
    bool attached_slot_done = false;   // N > 1: this rank's slot has been pulled in by its search kernel, the other slots are still on the host
    // reduction
    double* d_partials = nullptr;
    unsigned* d_done = nullptr;
    double* h_out = nullptr;    // pinned + mapped 160
    double* h_out_dev = nullptr;   // its device alias
    int max_blocks = 0;
    // knn query scratch
    float* d_q_d2 = nullptr;
    // stats
    long long launches = 0;
    float last_ms = 0.f;
    int last_launches = 0;
    int group = 4;
    int cells_search = LI_CELLS_SEARCH_DEFAULT;   // 1 shells on cells, 2 growing boxes, 3 growing boxes enumerate + stream (developer A/B: LIINIT_CELLS_SEARCH)
    bool cells_dynamic = false;       // cells search kernel with warp-granular dynamic scheduling (LIINIT_CELLS_SCHED=dynamic; not yet GPU-measured)
    unsigned* d_ticket = nullptr;
    bool cells_refresh_warp = true;   // directory refresh: warp per brick (false: thread per brick, the version the CPU checker runs)
    bool cells = false;   // knn_index = LIINIT_KNN_CELLS: per-brick cell directory + thread-per-point search (cells.cuh)
    float rho2 = 0.09f;   // squared seed radius of the 5-NN search
    // map assessment (liinit_assess_*, assess_kernels.cuh): the stored scans and the buffers of an evaluation, allocated by
    // liinit_assess_reserve
    struct Assess {
        long long cap = 0;   // points (0: not reserved)
        int max_scans = 0;
        long long n = 0;     // stored points
        int scans = 0, skipped = 0;
        long long last_q = -1;   // queries of the last evaluation (-1: none since the reserve) ...
        long long last_n = 0;    // ... and the stored points it placed
        float4* pts = nullptr;   // stored body points, w = scan index
        PoseD* poses = nullptr;
        float4* world = nullptr;   // placed points, stored order
        float4* sorted = nullptr;  // placed points in cell order, w = stored index
        unsigned long long* key = nullptr;
        unsigned long long* skey = nullptr;
        unsigned* k[2] = {nullptr, nullptr};   // one allocation of 2 N words: k[1] = k[0] + N
        unsigned* v[2] = {nullptr, nullptr};
        int* hist = nullptr;
        int* tc = nullptr;   // per-block counts: cell starts, queries, tasks
        int* tq = nullptr;
        int* tt = nullptr;
        int* cell_start = nullptr;
        unsigned long long* cell_key = nullptr;
        int* cell_q0 = nullptr;
        int* qlist = nullptr;
        int4* tasks = nullptr;
        int* qn = nullptr;
        double* qh = nullptr;
        double* qv = nullptr;
        int* box = nullptr;
        AsTotals* tot = nullptr;
        unsigned* ticket = nullptr;
        // timed store (liinit_assess_reserve_timed, assess_time_kernels.cuh): raw points by stored index (only a timed scan's are
        // used), per scan its pose table and prior state, the pose pool, and per scan the undistortion target of an evaluation
        bool timed = false;
        float4* raw = nullptr;
        AtScan* at = nullptr;
        PoseD* at_end = nullptr;
        double* pool = nullptr;
        long long pool_cap = 0, pool_rows = 0;   // pose rows
        int timed_scans = 0, untimed_scans = 0;
        long long hold_seq = -1;   // stage_seq of the held cloud (-1: no hold) ...
        int hold_n = 0;            // ... its points ...
        long long hold_at = 0;     // ... and the stored-point count it was copied behind
    } A;
    // LIO-phase replay (liinit_replay_*): sub-frames in the layout of the frame slots, appended in processing order
    struct ReplayFrame {
        double t_beg;
        float end_ms;
        int n;
        long long lo;   // first stored point
    };
    struct Replay {
        long long cap = 0, n = 0;   // points (cap 0: not reserved)
        int max_frames = 0, skipped = 0;
        float4* pts = nullptr;      // xyz, w = time [ms]
        float* inten = nullptr;
        std::vector<ReplayFrame> fr;
    } R;
    // map snapshot (liinit_map_snapshot / _restore): device copies of the map state and of the staged raw cloud, host copies of the
    // counters the host mirrors
    struct Snap {
        bool have = false;
        uint4* ent = nullptr;
        uint4* aux = nullptr;
        int* brick_slots = nullptr;
        unsigned long long* cocc = nullptr;
        unsigned short* cdir = nullptr;
        unsigned long long* sb_keys = nullptr;
        unsigned long long* sb_occ = nullptr;
        int* counters = nullptr;                // CNT_COUNT ints, then the pool top as one 8-byte word
        float4* pool = nullptr;
        unsigned long long pool_alloc = 0;      // points
        float4* stage_pts = nullptr;
        float4* stage_attr = nullptr;
        int stage_alloc = 0;                    // points
        int h_counters[CNT_COUNT] = {};
        unsigned long long pool_top = 0;
        int raw_n = 0;
        bool stage_attr_on = false;
    } snap;
    // replay sharing (liinit_replay_share): a worker reads its lead's replay store and map snapshot instead of its own; a lead counts
    // the workers that read its store and snapshot (while any does, neither may change or go away)
    Ctx* share_lead = nullptr;
    std::atomic<int> share_workers{0};
};

#define CU(call)                                                                                     \
    do {                                                                                             \
        cudaError_t _e = (call);                                                                     \
        if (_e != cudaSuccess) {                                                                     \
            c->err = std::string(#call) + ": " + cudaGetErrorString(_e);                             \
            return LIINIT_ERR_CUDA;                                                                  \
        }                                                                                            \
    } while (0)

inline int nblk(long long n, int t) { return (int)((n + t - 1) / t); }

// per-call device scratch that is released on every return path (the CU() macro returns early on a CUDA error)
template <class T>
struct DevBuf {
    T* p = nullptr;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { if (p) cudaFree(p); }
    cudaError_t alloc(size_t count) { return cudaMalloc(&p, count * sizeof(T)); }
};

int fail(Ctx* c, int code, const std::string& msg) {
    c->err = msg;
    return code;
}

// copy n points with a float stride from host to d_stage_pts[0..n) as float4
int stage_points(Ctx* c, const float* xyz, int stride, int n) {
    if (n > c->stage_pts_cap) return fail(c, LIINIT_ERR_CAPACITY, "batch exceeds staging capacity");
    c->raw_n = 0;   // the staging buffer is shared with the raw-scan front end
    c->stage_seq++;
    if (stride == 4) {
        CU(cudaMemcpyAsync(c->d_stage_pts, xyz, (size_t)n * 16, cudaMemcpyHostToDevice, c->stream));
        return LIINIT_OK;
    }
    if (stride != 3 && stride != 12) return fail(c, LIINIT_ERR_INVALID, "stride_floats must be 3, 4 or 12");
    size_t nf = (size_t)n * stride;
    if (nf > c->stage_raw_floats) return fail(c, LIINIT_ERR_CAPACITY, "batch exceeds raw staging capacity");
    CU(cudaMemcpyAsync(c->d_stage_raw, xyz, nf * 4, cudaMemcpyHostToDevice, c->stream));
    k_repack<<<nblk(n, 256), 256, 0, c->stream>>>(c->d_stage_raw, stride, n, c->d_stage_pts);
    c->launches++;
    CU(cudaGetLastError());
    return LIINIT_OK;
}

// ---- the device-pointer twins (liinit_*_device) ----
bool has_comm(const Ctx* c) {
#ifndef LI_SIMT_EMUL
    return c->comm != nullptr;
#else
    (void)c;
    return false;
#endif
}

// An argument of a device twin must be device (or managed) memory of the context's device. Checked before anything is changed.
int check_device_ptr(Ctx* c, const void* p, const char* what) {
    if (!p) return fail(c, LIINIT_ERR_INVALID, std::string(what) + " is null");
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
        cudaGetLastError();
        return fail(c, LIINIT_ERR_INVALID, std::string(what) + " is not a pointer the CUDA runtime knows");
    }
    if (at.type != cudaMemoryTypeDevice && at.type != cudaMemoryTypeManaged)
        return fail(c, LIINIT_ERR_INVALID, std::string(what) + " is not device memory (the host twin takes host memory)");
    if (at.device != c->device)
        return fail(c, LIINIT_ERR_INVALID, std::string(what) + " is memory of device " + std::to_string(at.device) + ", the context runs on device " +
                                               std::to_string(c->device));
    return LIINIT_OK;
}

int device_twin_check(Ctx* c, int stride) {
    if (has_comm(c)) return fail(c, LIINIT_ERR_INVALID, "the device-pointer entry points do not take a communicator (liinit_comm_init)");
    if (stride != 3 && stride != 4 && stride != 12) return fail(c, LIINIT_ERR_INVALID, "stride_floats must be 3, 4 or 12");
    return LIINIT_OK;
}

bool aligned16(const void* p) { return ((size_t)p & 15) == 0; }

// stage_points for device memory: a 16-byte aligned stride-4 batch is used in place, any other one is repacked into d_stage_pts
// straight from the caller's memory. *pts: where the batch now is, as float4.
int stage_points_device(Ctx* c, const float* xyz, int stride, int n, const float4** pts) {
    if (n > c->stage_pts_cap) return fail(c, LIINIT_ERR_CAPACITY, "batch exceeds staging capacity");
    c->raw_n = 0;   // as stage_points: the staging buffer is shared with the raw-scan front end
    c->stage_seq++;
    if (stride == 4 && aligned16(xyz)) {
        *pts = reinterpret_cast<const float4*>(xyz);
        return LIINIT_OK;
    }
    k_repack<<<nblk(n, 256), 256, 0, c->stream>>>(xyz, stride, n, c->d_stage_pts);
    c->launches++;
    CU(cudaGetLastError());
    *pts = c->d_stage_pts;
    return LIINIT_OK;
}

// the batch of the host (staging copy) or the device twin as float4
int stage_batch(Ctx* c, const float* xyz, int stride, int n, bool dev, const float4** pts) {
    if (dev) return stage_points_device(c, xyz, stride, n, pts);
    *pts = c->d_stage_pts;
    return stage_points(c, xyz, stride, n);
}

// the first n device points into packed host xyz [n*3] (synchronises)
int download_xyz(Ctx* c, const float4* src, size_t n, float* xyz) {
    std::vector<float4> b(n);
    CU(cudaMemcpyAsync(b.data(), src, n * sizeof(float4), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    for (size_t i = 0; i < n; i++) {
        xyz[3 * i] = b[i].x; xyz[3 * i + 1] = b[i].y; xyz[3 * i + 2] = b[i].z;
    }
    return LIINIT_OK;
}

int fetch_counters(Ctx* c) {
    CU(cudaMemcpyAsync(c->h_counters, c->d_counters, sizeof(int) * CNT_COUNT, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaMemcpyAsync(c->h_pool_top, c->M.pool_top, sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return LIINIT_OK;
}

// Capacity errors are reported ONCE, to the call that hit them: the bits are cleared on the device so that the calls after a box
// delete / a compaction are judged on their own (they used to stay set until the next Build).
int check_map_err(Ctx* c) {
    int e = c->h_counters[CNT_ERR];
    if (e & (ERR_HASH_FULL | ERR_POOL_FULL)) {
        cudaMemsetAsync(c->d_counters + CNT_ERR, 0, sizeof(int), c->stream);
        c->h_counters[CNT_ERR] = 0;
    }
    if (e & ERR_POOL_FULL) {
        // the failed reservations left the bump allocator beyond the capacity (k_ins_reserve): back to the end of the last slab in use
        const int nb = c->h_counters[CNT_BRICKS];
        cudaMemsetAsync(c->M.pool_top, 0, sizeof(unsigned long long), c->stream);
        if (nb > 0) {
            k_pool_top_recompute<<<nblk(nb, 256), 256, 0, c->stream>>>(c->M, nb);
            c->launches++;
        }
        cudaMemcpyAsync(c->h_pool_top, c->M.pool_top, sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->stream);
        cudaStreamSynchronize(c->stream);
    }
    if (e & ERR_HASH_FULL) return fail(c, LIINIT_ERR_CAPACITY, "brick hash table full (raise hash_capacity_log2 / max_map_points)");
    if (e & ERR_POOL_FULL) return fail(c, LIINIT_ERR_CAPACITY, "map point pool full (raise max_map_points, or liinit_map_compact after deletes)");
    return LIINIT_OK;
}

int reset_batch_counters(Ctx* c) {
    // touched, changed, nadd, nnod reset; err, live, bricks, dropped persist
    static const int zeros[CNT_COUNT] = {0};
    CU(cudaMemcpyAsync(c->d_counters + CNT_TOUCHED, zeros, sizeof(int), cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(c->d_counters + CNT_CHANGED, zeros, sizeof(int), cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(c->d_counters + CNT_COUPLED, zeros, sizeof(int), cudaMemcpyHostToDevice, c->stream));
    return LIINIT_OK;
}

// cell directory of the bricks the batch touched (after the commit / compaction that fixed their counts)
void refresh_cells_touched(Ctx* c) {
    if (!c->cells) return;
    if (c->cells_refresh_warp) k_cells_refresh_touched_warp<<<c->num_sms * 16, 128, 0, c->stream>>>(c->M);
    else k_cells_refresh_touched<<<c->num_sms * 8, 128, 0, c->stream>>>(c->M);
    c->launches++;
}

// plain insert of pts[0..n) (optionally only flag==want)
int plain_insert(Ctx* c, const float4* pts, int n, const int* sel, int want) {
    if (n <= 0) return LIINIT_OK;
    int r = reset_batch_counters(c);
    if (r) return r;
    k_ins_count<<<nblk(n, 256), 256, 0, c->stream>>>(c->M, pts, n, sel, want, c->d_slot_of);
    // the number of touched bricks is only known on the device: fixed grids, grid-stride loops inside
    const int gfix = c->num_sms * 8;
    k_ins_reserve<<<gfix, 256, 0, c->stream>>>(c->M);
    k_ins_append<<<nblk(n, 256), 256, 0, c->stream>>>(c->M, pts, n, c->d_slot_of);
    k_ins_commit<<<gfix, 256, 0, c->stream>>>(c->M);
    c->launches += 4;
    refresh_cells_touched(c);
    CU(cudaGetLastError());
    return LIINIT_OK;
}

// the temporary voxel hash, shrunk to the next power of two >= 2n slots (never beyond the allocation)
VoxTmp sized_vox(Ctx* c, int n) {
    VoxTmp V = c->V;
    unsigned m = 1024;
    while (m < 2u * (unsigned)n && m - 1 < c->V.mask) m <<= 1;
    if (m - 1 < V.mask) V.mask = m - 1;
    return V;
}

int downsample_insert(Ctx* c, const float4* pts, int n, const int* sel, int want) {
    if (n <= 0) return LIINIT_OK;
    int r = reset_batch_counters(c);
    if (r) return r;
    VoxTmp V = sized_vox(c, n);   // batch-sized temporary hash: clearing / walking 2M slots for a 10k-point batch is waste
    k_vox_clear<<<nblk((long long)V.mask + 1, 256), 256, 0, c->stream>>>(V);
    k_ds_link<<<nblk(n, 256), 256, 0, c->stream>>>(c->M, V, pts, n, sel, want, c->d_vslot_of, c->d_slot_of, c->d_ins);
    k_ins_reserve<<<c->num_sms * 8, 256, 0, c->stream>>>(c->M);
    k_ds_scan<<<nblk((long long)V.mask + 1, 128), 128, 0, c->stream>>>(c->M, V, pts, c->d_vslot_of);
    k_ds_replay<<<nblk((long long)V.mask + 1, 128), 128, 0, c->stream>>>(c->M, V, pts, c->d_vslot_of, c->d_ins);
    // boxes that share a point with another box of the batch (one-ulp overlaps of the float boxes): one warp, batch order (returns at once when there are none)
    k_ds_coupled<<<1, 32, 0, c->stream>>>(c->M, V, pts, c->d_vslot_of, c->d_ins, reinterpret_cast<int*>(c->d_rs_keys), reinterpret_cast<int*>(c->d_rs_vals));
    k_ds_append<<<nblk(n, 256), 256, 0, c->stream>>>(c->M, pts, n, c->d_slot_of, c->d_ins);
    // tombstoned bricks were added to the touched list by the replay (worst case n + n bricks): grid-stride inside
    k_ds_compact<<<c->num_sms * 8, 256, 0, c->stream>>>(c->M);
    c->launches += 8;
    refresh_cells_touched(c);
    CU(cudaGetLastError());
    return LIINIT_OK;
}

void fill_pose(PoseD& P, const double* R, const double* p, const double* RLI, const double* TLI) {
    memcpy(P.R, R, 72);
    memcpy(P.p, p, 24);
    memcpy(P.RLI, RLI, 72);
    memcpy(P.TLI, TLI, 24);
}

// An attached host scan that something other than the search kernel needs: pull it into d_body now.
void materialize_scan(Ctx* c) {
    if (!c->attached) return;
    if (c->attached_slot_done) {   // only what the search kernel did not read: the other ranks' slots [0, lo) and [lo + S.n, n)
        const int lo = c->shard_lo, hi = c->shard_lo + c->S.n;
        if (lo > 0) {
            k_repack<<<nblk(lo, 256), 256, 0, c->stream>>>(c->attached, c->attached_stride, lo, c->d_body);
            c->launches++;
        }
        if (hi < c->scan_n) {
            k_repack<<<nblk(c->scan_n - hi, 256), 256, 0, c->stream>>>(c->attached + (size_t)hi * c->attached_stride, c->attached_stride, c->scan_n - hi,
                                                                       c->d_body + hi);
            c->launches++;
        }
    } else {
        k_repack<<<nblk(c->scan_n, 256), 256, 0, c->stream>>>(c->attached, c->attached_stride, c->scan_n, c->d_body);
        c->launches++;
    }
    c->attached = nullptr;
    c->attached_slot_done = false;
}

// A new scan starts with nothing selected and no neighbours (Nearest_Points / point_selected_surf at iteration 0). The search
// pass that normally follows overwrites both arrays for every point of the scan, so the two fills are only issued when
// something else looks at them first (map_incremental, the download hooks): two stream operations fewer per scan.
int init_scan_state(Ctx* c) {
    if (!c->scan_fresh) return LIINIT_OK;
    CU(cudaMemsetAsync(c->d_selected, 0, (size_t)c->scan_n, c->stream));
    CU(cudaMemsetAsync(c->d_near_xyz, 0, (size_t)c->scan_n * 5 * sizeof(float4), c->stream));   // w = 0: no neighbour at any rank
    c->scan_fresh = false;
    return LIINIT_OK;
}

// A new frame of n points is resident (or attached): this rank's shard is [rank * cnt, rank * cnt + cnt) clipped to n with
// cnt = ceil(n / nranks) -- equal-sized slots, so that the per-point results can be all-gathered in place.
void set_scan(Ctx* c, int n) {
    c->scan_n = n;
    const int cnt = (n + c->nranks - 1) / c->nranks;
    int lo = c->rank * cnt;
    if (lo > n) lo = n;
    int hi = lo + cnt;
    if (hi > n) hi = n;
    c->shard_lo = lo;
    c->S.body = c->d_body + lo;
    c->S.world = c->d_world + lo;
    c->S.near_ids = c->d_near_ids + (size_t)lo * 5;
    c->S.near_xyz = c->d_near_xyz + (size_t)lo * 5;
    c->S.selected = c->d_selected + lo;
    c->S.normvec = c->d_normvec + lo;
    c->S.n = hi - lo;
    c->have_neighbors = false;
    c->scan_fresh = true;
    c->state_gathered = c->nranks == 1;
}

// Lanes per scan point when the caller left knn_group_lanes = 0. A warp works on 32/G points at once and lives as long as its slowest
// one: 4 lanes give the best throughput once every SM holds several such batches, but a small frame then occupies a fraction of the
// GPU for a long batch time. The thresholds come from a frame-size sweep of the search kernel (tools/probe_small.py, C2 scene) on the
// previous target GPU; one H100 run did not separate them from the alternatives beyond noise (DESIGN section 3). Every G gives the
// same neighbours.
int group_for(int n) {
    if (n <= 14000) return 32;
    if (n <= 70000) return 8;
    return 4;
}

// The search kernel of a pass reads an attached host frame in place: its own slot only. With one rank that is the whole frame and
// nothing is left to copy; with several the rest stays on the host until somebody needs the whole frame (materialize_scan).
const float* attached_slot(Ctx* c) {
    return (c->attached && !c->attached_slot_done) ? c->attached + (size_t)c->shard_lo * c->attached_stride : nullptr;
}
void attached_slot_read(Ctx* c) {
    if (c->nranks > 1 && c->S.n < c->scan_n) c->attached_slot_done = true;
    else c->attached = nullptr;
}

#ifndef LI_KNN_WAVES
#define LI_KNN_WAVES 6   // grid cap of the search kernel in resident waves (H100 sweep, DESIGN section 3: 1, 2, 4 and 8 were slower)
#endif
template <int G>
void launch_knn_scan(Ctx* c, const PoseD& P) {
    long long threads = (long long)c->S.n * G;
    int grid = nblk(threads, LI_KNN_THREADS);
    // Large frames: at most LI_KNN_WAVES waves of resident blocks, every warp strides over the query batches. The warps of the
    // first blocks then take one batch more than the rest and start first, and the blocks that start last are the short ones.
    const int cap = c->num_sms * LI_KNN_MIN_BLOCKS * LI_KNN_WAVES;
    if (grid > cap) grid = cap;
    // a later search pass of the same scan, no map point removed in between: seeded by the previous pass's neighbours (knn_kernels.cuh)
    const bool seeded = c->have_neighbors && !c->scan_fresh && c->nbr_epoch == c->map_epoch && c->reseed;
    if (const float* raw = attached_slot(c)) {
        k_knn_scan<G, true><<<grid, LI_KNN_THREADS, 0, c->stream>>>(c->M, c->S, P, c->rho2, raw, c->attached_stride);
        attached_slot_read(c);   // the kernel leaves the packed copy in d_body
    } else if (seeded) {
        k_knn_scan<G, false, true><<<grid, LI_KNN_THREADS, 0, c->stream>>>(c->M, c->S, P, c->rho2, nullptr, 0);
    } else {
        k_knn_scan<G, false><<<grid, LI_KNN_THREADS, 0, c->stream>>>(c->M, c->S, P, c->rho2, nullptr, 0);
    }
}

#ifndef LI_PLANE_WAVES
#define LI_PLANE_WAVES 1   // the plane pass runs LI_PLANE_WAVES x (2 blocks per SM); each thread strides over the scan
#endif

template <int MINB, int SEARCH>
void launch_knn_cells_scan_t(Ctx* c, const PoseD& P) {
    if (c->cells_dynamic) {   // persistent grid, warps pull 32-point batches from a ticket counter (reset in stream order)
        cudaMemsetAsync(c->d_ticket, 0, sizeof(unsigned), c->stream);
        const int pgrid = c->num_sms * MINB;
        if (const float* raw = attached_slot(c)) {
            k_knn_cells_scan_dyn<true, MINB, SEARCH><<<pgrid, LI_CELLS_THREADS, 0, c->stream>>>(c->M, c->S, P, c->rho2, raw, c->attached_stride, c->d_ticket);
            attached_slot_read(c);
        } else {
            k_knn_cells_scan_dyn<false, MINB, SEARCH><<<pgrid, LI_CELLS_THREADS, 0, c->stream>>>(c->M, c->S, P, c->rho2, nullptr, 0, c->d_ticket);
        }
        return;
    }
    const int grid = nblk(c->S.n, LI_CELLS_THREADS);
    if (const float* raw = attached_slot(c)) {
        k_knn_cells_scan<true, MINB, SEARCH><<<grid, LI_CELLS_THREADS, 0, c->stream>>>(c->M, c->S, P, c->rho2, raw, c->attached_stride);
        attached_slot_read(c);   // the kernel leaves the packed copy in d_body
    } else {
        k_knn_cells_scan<false, MINB, SEARCH><<<grid, LI_CELLS_THREADS, 0, c->stream>>>(c->M, c->S, P, c->rho2, nullptr, 0);
    }
}
// LI_CELLS_MINB (resident blocks per SM the kernel is compiled for): 6 -> 80 registers; 4 (more registers) and 8 (spills) were slower
void launch_knn_cells_scan(Ctx* c, const PoseD& P) {
    if (c->cells_search == 1) launch_knn_cells_scan_t<LI_CELLS_MINB, 1>(c, P);
    else if (c->cells_search == 2) launch_knn_cells_scan_t<LI_CELLS_MINB, 2>(c, P);
    else launch_knn_cells_scan_t<LI_CELLS_MINB, 3>(c, P);
}

template <bool IMU, bool SEARCH>
void launch_plane(Ctx* c, const PoseD& P, double* out) {
    // one wave of 256-thread blocks (2 resident per SM at ~100-130 registers), grid-stride over the scan
    int grid = nblk(c->S.n, 256);
    if (grid > c->num_sms * LI_PLANE_MIN_BLOCKS * LI_PLANE_WAVES) grid = c->num_sms * LI_PLANE_MIN_BLOCKS * LI_PLANE_WAVES;
    if (grid < 1) grid = 1;   // (an empty slot of a multi-GPU frame still takes part in the exchange)
    const XchgTable* X = (c->nranks > 1 && c->comm_p2p) ? c->d_xtab : nullptr;
    // the lockstep search leaves the neighbour copies in S.near_xyz itself; the cell-directory search hands pool offsets over, which
    // the plane kernel of that pass gathers (and leaves as copies); a reuse pass reads the copies
    if (SEARCH && c->cells) k_icp_plane<IMU, SEARCH, true><<<grid, 256, 0, c->stream>>>(c->M, c->S, P, c->d_partials, c->d_done, out, X, c->xseq);
    else k_icp_plane<IMU, SEARCH, false><<<grid, 256, 0, c->stream>>>(c->M, c->S, P, c->d_partials, c->d_done, out, X, c->xseq);
}

// out: where the last block of the plane kernel leaves the 160-double result block -- the caller's device buffer
// (liinit_icp_iterate_device) or the device alias of the context's page-locked host block (liinit_icp_iterate: the
// kernel writes the 1.28 kB over PCIe itself, no copy operation behind it).
int run_pass(Ctx* c, const double* R, const double* p, const double* RLI, const double* TLI, int imu_en, int search, double* out) {
    if (c->scan_n <= 0) return fail(c, LIINIT_ERR_INVALID, "no scan uploaded");
    if (!search && !c->have_neighbors) return fail(c, LIINIT_ERR_INVALID, "reuse pass before any search pass");
    PoseD P;
    fill_pose(P, R, p, RLI, TLI);
    double* const final_out = out;
    if (c->nranks > 1 && !c->comm_p2p) out = c->d_acc;   // NCCL mode: this rank's block; the sum over the ranks goes to final_out below
    if (c->nranks > 1) c->xseq++;                          // peer-memory mode: the plane kernel's last block sums over the ranks itself
    CU(cudaEventRecord(c->ev0, c->stream));
    if (search) {
        if (c->S.n == 0) {
            // an empty slot (more ranks than points): nothing to search
        } else if (c->cells) launch_knn_cells_scan(c, P);
        else switch (c->group ? c->group : group_for(c->S.n)) {
            case 16: launch_knn_scan<16>(c, P); break;
            case 32: launch_knn_scan<32>(c, P); break;
            case 2: launch_knn_scan<2>(c, P); break;
            case 8: launch_knn_scan<8>(c, P); break;
            default: launch_knn_scan<4>(c, P); break;
        }
        CU(cudaEventRecord(c->evm, c->stream));
        if (imu_en) launch_plane<true, true>(c, P, out); else launch_plane<false, true>(c, P, out);
        c->have_neighbors = true;
        c->nbr_epoch = c->map_epoch;
        c->scan_fresh = false;   // the two kernels wrote the neighbour copies / selected for every point of the scan
        c->launches += 2;
        c->last_launches = 2;
        c->last_was_search = true;
    } else {
        if (imu_en) launch_plane<true, false>(c, P, out); else launch_plane<false, false>(c, P, out);
        c->launches += 1;
        c->last_launches = 1;
        c->last_was_search = false;
    }
    CU(cudaEventRecord(c->ev1, c->stream));
    CU(cudaGetLastError());
    c->state_gathered = c->nranks == 1;
#ifndef LI_SIMT_EMUL
    if (c->nranks > 1 && !c->comm_p2p) {
        // the one exchange of the path (SURVEY.md section 8e): sum of [HtH 144 | Htr 12 | res_sq | m | pad 2] over the ranks, on the
        // context's stream, then to wherever the caller wants the block (page-locked host block or its own device buffer)
        NcclApi* N = nccl_api();
        ncclResult_t nr = N->AllReduce(c->d_acc, c->d_red, 160, ncclDouble, ncclSum, c->comm, c->stream);
        if (nr != ncclSuccess) return fail(c, LIINIT_ERR_CUDA, std::string("ncclAllReduce: ") + N->GetErrorString(nr));
        CU(cudaMemcpyAsync(final_out, c->d_red, 160 * sizeof(double), cudaMemcpyDefault, c->stream));
    }
#endif
    return LIINIT_OK;
}

#ifndef LI_SIMT_EMUL
// In-place all-gather of one per-point array (elem bytes per point) over the equal-sized shard slots.
int gather_array(Ctx* c, void* base, size_t elem) {
    NcclApi* N = nccl_api();
    const int cnt = (c->scan_n + c->nranks - 1) / c->nranks;
    const size_t bytes = (size_t)cnt * elem;
    ncclResult_t nr = N->AllGather((const char*)base + (size_t)c->rank * bytes, base, bytes, ncclChar, c->comm, c->stream);
    if (nr != ncclSuccess) return fail(c, LIINIT_ERR_CUDA, std::string("ncclAllGather: ") + N->GetErrorString(nr));
    return LIINIT_OK;
}
#endif

// N > 1: bring the other ranks' per-point results (Nearest_Points, flags, normals, world points) onto this device. Collective:
// every rank makes the same call (liinit_map_incremental and the download hooks do).
int gather_scan_state(Ctx* c) {
    if (c->state_gathered) return LIINIT_OK;
#ifndef LI_SIMT_EMUL
    int r;
    if ((r = gather_array(c, c->d_near_xyz, 5 * sizeof(float4)))) return r;
    if ((r = gather_array(c, c->d_selected, 1))) return r;
    if ((r = gather_array(c, c->d_normvec, sizeof(float4)))) return r;
    if ((r = gather_array(c, c->d_world, sizeof(float4)))) return r;
#endif
    c->state_gathered = true;
    return LIINIT_OK;
}

// One stable 8-bit pass of the radix sort (sort_kernels.cuh) of the pairs (k[cur], v[cur]) into (k[cur ^ 1], v[cur ^ 1]); cur then names
// the sorted pairs. n: the element count, or the bound the launch is sized for when n_dev holds the count on the device.
void rs_pass(Ctx* c, unsigned* const k[2], unsigned* const v[2], int& cur, int* hist, int n, const int* n_dev, int shift) {
    const int ntiles = nblk(n, RS_TILE);
    k_rs_hist<<<nblk(ntiles, 4), 128, 0, c->stream>>>(k[cur], n, n_dev, shift, ntiles, hist);
    k_rs_scan<<<1, 1024, 0, c->stream>>>(256 * ntiles, hist);
    k_rs_scatter<<<nblk(ntiles, 4), 128, 0, c->stream>>>(k[cur], v[cur], n, n_dev, shift, ntiles, hist, k[cur ^ 1], v[cur ^ 1]);
    c->launches += 3;
    cur ^= 1;
}

// ---- cut-frame preprocess ------------------------------------------------------------------------------------------------
void frame_free(Ctx* c) {
    cudaFree(c->d_fr_in); cudaFree(c->d_fr_dec); cudaFree(c->d_fr_inten); cudaFree(c->d_fr_flag); cudaFree(c->d_fr_keys); cudaFree(c->d_fr_vals);
    cudaFree(c->d_fr_aux); cudaFree(c->d_fr_yaw); cudaFree(c->d_fr_tsum); cudaFree(c->d_fr_ring); cudaFree(c->d_fr_tab); cudaFreeHost(c->h_fr_tab);
    cudaFree(c->d_fr_slot_pts); cudaFree(c->d_fr_slot_inten);
    c->d_fr_in = nullptr; c->d_fr_dec = nullptr; c->d_fr_inten = nullptr; c->d_fr_flag = nullptr; c->d_fr_keys = nullptr; c->d_fr_vals = nullptr;
    c->d_fr_aux = nullptr; c->d_fr_yaw = nullptr; c->d_fr_tsum = nullptr; c->d_fr_ring = nullptr; c->d_fr_tab = nullptr; c->h_fr_tab = nullptr;
    c->d_fr_slot_pts = nullptr; c->d_fr_slot_inten = nullptr;
    c->fr_in_bytes = 0;
    c->fr_ready = false;
}

int frame_tiles(Ctx* c) { return nblk(c->stage_pts_cap, LI_FR_TILE); }

// buffers of the cut, sized for stage_pts_cap points (the input buffer grows with the largest message seen)
int frame_alloc(Ctx* c, size_t in_bytes) {
    if (!c->fr_ready) {
        const size_t cap = (size_t)c->stage_pts_cap;
        cudaError_t e = cudaSuccess;
        auto A = [&](void** p, size_t bytes) { if (e == cudaSuccess) e = cudaMalloc(p, bytes); };
        A((void**)&c->d_fr_dec, cap * sizeof(float4));
        A((void**)&c->d_fr_inten, cap * sizeof(float));
        A((void**)&c->d_fr_flag, cap * sizeof(int));
        A((void**)&c->d_fr_keys, cap * sizeof(unsigned));
        A((void**)&c->d_fr_vals, cap * sizeof(unsigned));
        A((void**)&c->d_fr_aux, cap * sizeof(unsigned));
        A((void**)&c->d_fr_yaw, cap * sizeof(double));
        A((void**)&c->d_fr_tsum, (size_t)2 * frame_tiles(c) * sizeof(int));
        A((void**)&c->d_fr_ring, 513 * sizeof(int));
        A((void**)&c->d_fr_tab, sizeof(FrameTable));
        A((void**)&c->d_fr_slot_pts, LIINIT_FRAME_SLOTS * cap * sizeof(float4));
        A((void**)&c->d_fr_slot_inten, LIINIT_FRAME_SLOTS * cap * sizeof(float));
        if (e == cudaSuccess) e = cudaMallocHost((void**)&c->h_fr_tab, sizeof(FrameTable));
        if (e != cudaSuccess) {
            frame_free(c);
            c->err = std::string("frame buffers: ") + cudaGetErrorString(e);
            return LIINIT_ERR_CUDA;
        }
        for (int s = 0; s < LIINIT_FRAME_SLOTS; s++) {
            c->fr_slot_seq[s] = -1;
            c->fr_slot_nsub[s] = 0;
        }
        c->fr_ready = true;
    }
    if (in_bytes > c->fr_in_bytes) {
        CU(cudaStreamSynchronize(c->stream));
        cudaFree(c->d_fr_in);
        c->d_fr_in = nullptr;
        c->fr_in_bytes = 0;
        CU(cudaMalloc(&c->d_fr_in, in_bytes));
        c->fr_in_bytes = in_bytes;
    }
    return LIINIT_OK;
}

// argument checks shared by both message types; R = required_cut_num
int frame_check(Ctx* c, const liinit_frame_params* p, int n, int cap, bool pcl2, int* R) {
    const int t = p->lidar_type;
    if (pcl2 ? !(t == LIINIT_LIDAR_VELO || t == LIINIT_LIDAR_OUSTER || t == LIINIT_LIDAR_PANDAR || t == LIINIT_LIDAR_ROBOSENSE) : t != LIINIT_LIDAR_AVIA)
        return fail(c, LIINIT_ERR_INVALID, "lidar_type does not match the message type");
    if (p->point_filter_num <= 0 || p->required_frame_num <= 0 || p->required_frame_num > LIINIT_FRAME_MAX_CUT)
        return fail(c, LIINIT_ERR_INVALID, "point_filter_num must be positive and required_frame_num in [1, LIINIT_FRAME_MAX_CUT]");
    if (n > c->stage_pts_cap) return fail(c, LIINIT_ERR_CAPACITY, "message exceeds the raw staging capacity");
    *R = p->scan_count < (pcl2 ? 20 : 5) ? 1 : p->required_frame_num;
    if (n > 0 && cap < *R) return fail(c, LIINIT_ERR_CAPACITY, "cap is smaller than required_cut_num");
    return LIINIT_OK;
}

// flags and decoded points are in place, tsum holds the per-block flag counts: compaction, time sort, cut, gather, table
int frame_finish(Ctx* c, int n, int R, double S, int* tsum, liinit_subframe* out, int* n_sub) {
    const int nb = nblk(n, LI_FR_TILE);
    k_rs_scan<<<1, 1024, 0, c->stream>>>(nb, tsum);
    k_fr_compact<<<nb, LI_FR_TILE, 0, c->stream>>>(c->d_fr_flag, n, tsum, c->d_fr_dec, nullptr, c->d_fr_keys, c->d_fr_vals, &c->d_fr_tab->V);
    unsigned* const k[2] = {c->d_fr_keys, c->d_rs_keys};
    unsigned* const v[2] = {c->d_fr_vals, c->d_rs_vals};
    int cur = 0;
    for (int pass = 0; pass < 4; pass++) rs_pass(c, k, v, cur, c->d_rs_hist, n, &c->d_fr_tab->V, 8 * pass);
    const int slot = (int)(c->fr_seq % LIINIT_FRAME_SLOTS);
    const size_t cap = (size_t)c->stage_pts_cap;
    k_fr_bounds<<<1, 32, 0, c->stream>>>(v[cur], c->d_fr_dec, R, S, c->d_fr_tab);
    k_fr_gather<<<nblk(n, 256), 256, 0, c->stream>>>(v[cur], c->d_fr_dec, c->d_fr_inten, S, c->d_fr_tab, c->d_fr_slot_pts + slot * cap,
                                                     c->d_fr_slot_inten + slot * cap);
    c->launches += 4;
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(c->h_fr_tab, c->d_fr_tab, offsetof(FrameTable, sub) + (size_t)R * sizeof(FrameSub), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    const FrameTable* T = c->h_fr_tab;
    if (T->err & 1) return fail(c, LIINIT_ERR_INVALID, "ring >= 128 in the constant-rotation model");
    *n_sub = T->nsub;
    if (T->nsub == 0) return LIINIT_OK;
    c->fr_slot_seq[slot] = c->fr_seq;
    c->fr_slot_nsub[slot] = T->nsub;
    for (int k = 0; k < T->nsub; k++) {
        c->fr_slot_sub[slot][k] = T->sub[k];
        out[k].handle = c->fr_seq * LIINIT_FRAME_MAX_CUT + k;
        out[k].t_beg = T->sub[k].lfet / double(1000);
        out[k].end_ms = T->sub[k].end_ms;
        out[k].n = T->sub[k].n;
    }
    c->fr_seq++;
    return LIINIT_OK;
}

// the sub-frame a handle names, or nullptr when its slot has been reused
const FrameSub* frame_lookup(Ctx* c, long long handle, int* slot) {
    if (!c->fr_ready || handle < 0) return nullptr;
    const long long seq = handle / LIINIT_FRAME_MAX_CUT;
    const int k = (int)(handle % LIINIT_FRAME_MAX_CUT);
    const int s = (int)(seq % LIINIT_FRAME_SLOTS);
    if (c->fr_slot_seq[s] != seq || k >= c->fr_slot_nsub[s]) return nullptr;
    *slot = s;
    return &c->fr_slot_sub[s][k];
}

void assess_free(Ctx* c) {
    Ctx::Assess& A = c->A;
    cudaFree(A.pts); cudaFree(A.poses); cudaFree(A.world); cudaFree(A.sorted); cudaFree(A.key); cudaFree(A.skey);
    cudaFree(A.k[0]); cudaFree(A.v[0]); cudaFree(A.v[1]); cudaFree(A.hist); cudaFree(A.tc); cudaFree(A.tq); cudaFree(A.tt);
    cudaFree(A.cell_start); cudaFree(A.cell_key); cudaFree(A.cell_q0); cudaFree(A.qlist); cudaFree(A.tasks); cudaFree(A.qn); cudaFree(A.qh);
    cudaFree(A.qv); cudaFree(A.box); cudaFree(A.tot); cudaFree(A.ticket);
    cudaFree(A.raw); cudaFree(A.at); cudaFree(A.at_end); cudaFree(A.pool);
    A = Ctx::Assess{};
}

void replay_free(Ctx* c) {
    cudaFree(c->R.pts); cudaFree(c->R.inten);
    c->R = Ctx::Replay{};
}

void snap_free(Ctx* c) {
    Ctx::Snap& S = c->snap;
    cudaFree(S.ent); cudaFree(S.aux); cudaFree(S.brick_slots); cudaFree(S.cocc); cudaFree(S.cdir); cudaFree(S.sb_keys); cudaFree(S.sb_occ);
    cudaFree(S.counters); cudaFree(S.pool); cudaFree(S.stage_pts); cudaFree(S.stage_attr);
    S = Ctx::Snap{};
}

}  // namespace

struct liinit_ctx {
    Ctx c;
};

extern "C" {

const char* liinit_last_error(const liinit_ctx* h) { return h ? h->c.err.c_str() : g_create_error.c_str(); }

int liinit_create(const liinit_config* cfg, liinit_ctx** out) {
    if (!cfg || !out) {
        g_create_error = "null argument";
        return LIINIT_ERR_INVALID;
    }
    *out = nullptr;
    if (!(cfg->filter_size_map > 0.f) || cfg->max_map_points <= 0 || cfg->max_scan_points <= 0) {
        g_create_error = "filter_size_map, max_map_points and max_scan_points must be positive";
        return LIINIT_ERR_INVALID;
    }
    liinit_ctx* h = new liinit_ctx();
    Ctx* c = &h->c;
    c->cfg = *cfg;
    auto bail = [&](int code) {
        g_create_error = c->err;
        liinit_destroy(h);
        return code;
    };
#define CUC(call)                                                                 \
    do {                                                                          \
        cudaError_t _e = (call);                                                  \
        if (_e != cudaSuccess) {                                                  \
            c->err = std::string(#call) + ": " + cudaGetErrorString(_e);          \
            return bail(LIINIT_ERR_CUDA);                                         \
        }                                                                         \
    } while (0)
    int ndev = 0;
    CUC(cudaGetDeviceCount(&ndev));
    if (cfg->device_id < 0 || cfg->device_id >= ndev) {
        c->err = "device_id out of range (no usable CUDA device; there is no CPU fallback)";
        return bail(LIINIT_ERR_CUDA);
    }
    c->device = cfg->device_id;
    CUC(cudaSetDevice(c->device));
    cudaDeviceProp prop;
    CUC(cudaGetDeviceProperties(&prop, c->device));
    c->num_sms = prop.multiProcessorCount;
    CUC(cudaStreamCreateWithFlags(&c->own_stream, cudaStreamNonBlocking));
    c->stream = c->own_stream;
    CUC(cudaEventCreate(&c->ev0));
    CUC(cudaEventCreate(&c->ev1));
    CUC(cudaEventCreate(&c->evm));

    int bs = cfg->brick_cells_log2 > 0 ? cfg->brick_cells_log2 : 3;
    if (bs < 1 || bs > 4) {
        c->err = "brick_cells_log2 must be in [1,4]";
        return bail(LIINIT_ERR_INVALID);
    }
    int hl = cfg->hash_capacity_log2;
    if (hl <= 0) {
        // ~ one brick per 4 live points worst case for surface maps, load factor <= 0.5
        long long want = (long long)cfg->max_map_points / 2;
        hl = 16;
        while ((1ll << hl) < want && hl < 28) hl++;
    }
    if (hl < 10 || hl > 30) {
        c->err = "hash_capacity_log2 out of range";
        return bail(LIINIT_ERR_INVALID);
    }
    c->hash_slots = 1u << hl;
    // lanes per scan point of the lockstep search: fixed by the caller, or (0) chosen per pass from the frame size (group_for)
    c->group = (cfg->knn_group_lanes == 2 || cfg->knn_group_lanes == 4 || cfg->knn_group_lanes == 8 || cfg->knn_group_lanes == 16 || cfg->knn_group_lanes == 32) ? cfg->knn_group_lanes : 0;
    {
        const char* ge = getenv("LIINIT_KNN_GROUP");   // developer A/B
        if (ge && (atoi(ge) == 2 || atoi(ge) == 4 || atoi(ge) == 8 || atoi(ge) == 16 || atoi(ge) == 32)) c->group = atoi(ge);
    }

    {
        int ki = cfg->knn_index;
        if (ki == 0) {
            // developer A/B switch: run an unmodified caller (tests, bench) against the other index
            const char* e = getenv("LIINIT_KNN_INDEX");
            ki = (e && *e) ? atoi(e) : LIINIT_KNN_DEFAULT;
        }
        if (ki != LIINIT_KNN_BRICKS && ki != LIINIT_KNN_CELLS) {
            c->err = "knn_index must be 0, LIINIT_KNN_BRICKS or LIINIT_KNN_CELLS";
            return bail(LIINIT_ERR_INVALID);
        }
        // the cell directory is defined for 8x8x8-voxel bricks; another brick size keeps the brick search
        c->cells = ki == LIINIT_KNN_CELLS && bs == LI_CELLS_BSHIFT;
        const char* sd = getenv("LIINIT_CELLS_SCHED");
        if (sd && !strcmp(sd, "dynamic")) c->cells_dynamic = true;
        const char* rf = getenv("LIINIT_CELLS_REFRESH");
        if (rf && !strcmp(rf, "thread")) c->cells_refresh_warp = false;
        const char* cs = getenv("LIINIT_CELLS_SEARCH");
        if (cs && atoi(cs) >= 1 && atoi(cs) <= 3) c->cells_search = atoi(cs);
    }
    {
        float cells = cfg->knn_seed_radius_cells > 0.f ? cfg->knn_seed_radius_cells : 2.0f;
        float rho = cells * cfg->filter_size_map;
        c->rho2 = rho * rho;
    }
    MapDev& M = c->M;
    M.mask = c->hash_slots - 1;
    M.ds = cfg->filter_size_map;
    M.bshift = bs;
    // slabs grow geometrically and old slabs are abandoned: 3x live capacity + per-brick minimum slack
    unsigned long long pool = (unsigned long long)cfg->max_map_points * 3ull + (1ull << 20);
    if (pool > 0x7fffff00ull) pool = 0x7fffff00ull;   // ids are int32 pool offsets
    M.pool_cap = pool;
    CUC(cudaMalloc(&M.ent, (size_t)c->hash_slots * sizeof(uint4)));
    CUC(cudaMalloc(&M.brick_slots, (size_t)c->hash_slots * sizeof(int)));
    CUC(cudaMalloc(&M.aux, (size_t)c->hash_slots * sizeof(uint4)));
    CUC(cudaMalloc(&M.pool, (size_t)pool * sizeof(float4)));
    CUC(cudaMalloc(&M.pool_top, sizeof(unsigned long long)));
    M.cocc = nullptr;
    M.cdir = nullptr;
    M.sb_keys = nullptr;
    M.sb_occ = nullptr;
    M.sb_mask = 0;
    if (c->cells) {
        CUC(cudaMalloc(&M.cocc, (size_t)c->hash_slots * sizeof(unsigned long long)));
        CUC(cudaMalloc(&M.cdir, (size_t)c->hash_slots * 64 * sizeof(unsigned short)));
        // one super-brick per brick in the worst case (scattered points): same slot count as the brick hash
        M.sb_mask = c->hash_slots - 1;
        CUC(cudaMalloc(&M.sb_keys, (size_t)c->hash_slots * sizeof(unsigned long long)));
        CUC(cudaMalloc(&M.sb_occ, (size_t)c->hash_slots * sizeof(unsigned long long)));
        CUC(cudaMalloc(&c->d_ticket, sizeof(unsigned)));
    }
    int batch = cfg->max_scan_points > (1 << 20) ? cfg->max_scan_points : (1 << 20);
    c->stage_pts_cap = batch;
    CUC(cudaMalloc(&M.touched_list, (size_t)batch * 2 * sizeof(int)));
    CUC(cudaMalloc(&c->d_counters, sizeof(int) * CNT_COUNT));
    M.counters = c->d_counters;
    CUC(cudaMallocHost(&c->h_counters, sizeof(int) * CNT_COUNT));
    CUC(cudaMallocHost(&c->h_pool_top, sizeof(unsigned long long)));
    *c->h_pool_top = 0;
    c->stage_raw_floats = (size_t)batch * 12;
    CUC(cudaMalloc(&c->d_stage_raw, c->stage_raw_floats * 4));
    CUC(cudaMalloc(&c->d_stage_pts, (size_t)batch * sizeof(float4)));
    CUC(cudaMalloc(&c->d_stage_attr, (size_t)batch * sizeof(float4)));
    CUC(cudaMalloc(&c->d_slot_of, (size_t)batch * sizeof(int)));
    CUC(cudaMalloc(&c->d_vslot_of, (size_t)batch * sizeof(int)));
    CUC(cudaMalloc(&c->d_flag, (size_t)batch * sizeof(int)));
    CUC(cudaMalloc(&c->d_ins, (size_t)batch * sizeof(int)));
    CUC(cudaMalloc(&c->d_q_d2, (size_t)batch * 5 * sizeof(float)));
    {
        int vl = 10;
        while ((1ll << vl) < 2ll * batch) vl++;
        c->V.mask = (1u << vl) - 1;
        CUC(cudaMalloc(&c->V.keys, ((size_t)c->V.mask + 1) * 8));
        CUC(cudaMalloc(&c->V.head, ((size_t)c->V.mask + 1) * 4));
        CUC(cudaMalloc(&c->V.coupled, ((size_t)c->V.mask + 1) * 4));
        CUC(cudaMalloc(&c->V.sum, ((size_t)c->V.mask + 1) * sizeof(int4)));
        CUC(cudaMalloc(&c->V.clist, ((size_t)c->V.mask + 1) * 4));
        CUC(cudaMalloc(&c->d_vg_imin, ((size_t)c->V.mask + 1) * 4));
        CUC(cudaMalloc(&c->d_vg_block, ((size_t)batch / 1024 + 2) * 4));
        CUC(cudaMalloc(&c->d_vg_misc, 8 * 4));
        CUC(cudaMalloc(&c->d_rs_keys, (size_t)batch * 4));
        CUC(cudaMalloc(&c->d_rs_vals, (size_t)batch * 4));
        CUC(cudaMalloc(&c->d_rs_hist, ((size_t)batch / RS_TILE + 2) * 256 * 4));
        CUC(cudaMalloc(&c->d_vg_params, sizeof(VgParams)));
        CUC(cudaMalloc(&c->d_tmin_idx, 8));
        CUC(cudaMalloc(&c->d_poses, LIINIT_MAX_IMU_POSES * LI_POSE6D_DOUBLES * sizeof(double)));
    }
    int ns = cfg->max_scan_points + 64;   // (+ slack: equal-sized shard slots of a frame cut over up to 64 ranks)
    CUC(cudaMalloc(&c->d_acc, 160 * sizeof(double)));
    CUC(cudaMalloc(&c->d_red, 160 * sizeof(double)));
    CUC(cudaMalloc(&c->d_body, (size_t)ns * sizeof(float4)));
    CUC(cudaMalloc(&c->d_body_attr, (size_t)ns * sizeof(float4)));
    CUC(cudaMalloc(&c->d_world, (size_t)ns * sizeof(float4)));
    CUC(cudaMalloc(&c->d_near_ids, (size_t)batch * 5 * sizeof(int)));
    CUC(cudaMalloc(&c->d_near_xyz, (size_t)ns * 5 * sizeof(float4)));
    CUC(cudaMalloc(&c->d_selected, (size_t)ns));
    CUC(cudaMalloc(&c->d_normvec, (size_t)ns * sizeof(float4)));
    c->max_blocks = c->num_sms * 16;
    CUC(cudaMalloc(&c->d_partials, (size_t)c->max_blocks * 96 * sizeof(double)));
    CUC(cudaMalloc(&c->d_done, sizeof(unsigned)));
    CUC(cudaHostAlloc(&c->h_out, 160 * sizeof(double), cudaHostAllocMapped));
    CUC(cudaHostGetDevicePointer((void**)&c->h_out_dev, c->h_out, 0));
    CUC(cudaMemsetAsync(c->d_done, 0, sizeof(unsigned), c->stream));
    CUC(cudaMemsetAsync(c->d_counters, 0, sizeof(int) * CNT_COUNT, c->stream));
    CUC(cudaMemsetAsync(M.pool_top, 0, sizeof(unsigned long long), c->stream));
    k_map_clear<<<nblk(c->hash_slots, 256), 256, 0, c->stream>>>(M.ent, M.aux, c->hash_slots);
    c->launches++;
    if (c->cells) {
        k_sb_clear<<<nblk(c->hash_slots, 256), 256, 0, c->stream>>>(M);
        c->launches++;
    }
    CUC(cudaGetLastError());
    CUC(cudaStreamSynchronize(c->stream));
    c->S.body = c->d_body;
    c->S.world = c->d_world;
    c->S.near_ids = c->d_near_ids;
    c->S.near_xyz = c->d_near_xyz;
    c->S.selected = c->d_selected;
    c->S.normvec = c->d_normvec;
    c->S.n = 0;
#undef CUC
    *out = h;
    return LIINIT_OK;
}

int liinit_destroy(liinit_ctx* h) {
    if (!h) return LIINIT_OK;
    Ctx* c = &h->c;
    if (c->share_workers.load() > 0)
        return fail(c, LIINIT_ERR_INVALID, "workers share this context's replay store and map snapshot (liinit_replay_unshare them first)");
    cudaSetDevice(c->device);
    if (c->share_lead) {
        cudaStreamSynchronize(c->stream);   // its last reads of the lead's store and snapshot are done
        c->share_lead->share_workers--;
        c->share_lead = nullptr;
    }
    if (c->own_stream) cudaStreamSynchronize(c->own_stream);
    cudaFree(c->M.ent); cudaFree(c->M.brick_slots); cudaFree(c->M.aux); cudaFree(c->M.pool); cudaFree(c->M.pool_top); cudaFree(c->M.touched_list); cudaFree(c->M.cocc); cudaFree(c->M.cdir); cudaFree(c->M.sb_keys); cudaFree(c->M.sb_occ); cudaFree(c->d_ticket);
    cudaFree(c->d_counters); cudaFreeHost(c->h_counters); cudaFreeHost(c->h_pool_top); cudaFree(c->d_stage_raw); cudaFree(c->d_stage_pts);
    cudaFree(c->d_slot_of); cudaFree(c->d_vslot_of); cudaFree(c->d_flag); cudaFree(c->d_ins); cudaFree(c->V.keys); cudaFree(c->V.head); cudaFree(c->V.coupled); cudaFree(c->V.sum); cudaFree(c->V.clist); cudaFree(c->d_vg_imin); cudaFree(c->d_vg_block); cudaFree(c->d_vg_misc); cudaFree(c->d_rs_keys); cudaFree(c->d_rs_vals); cudaFree(c->d_rs_hist); cudaFree(c->d_vg_params); cudaFree(c->d_tmin_idx); cudaFree(c->d_poses);
    cudaFree(c->d_stage_attr); cudaFree(c->d_body_attr);
    cudaFree(c->d_body); cudaFree(c->d_world); cudaFree(c->d_near_ids); cudaFree(c->d_near_xyz); cudaFree(c->d_selected); cudaFree(c->d_normvec);
    cudaFree(c->d_acc); cudaFree(c->d_red);
#ifndef LI_SIMT_EMUL
    for (int r = 0; r < LI_MAX_RANKS; r++)
        if (c->peer_map[r]) cudaIpcCloseMemHandle(c->peer_map[r]);
    cudaFree(c->d_xtab);
    cudaFree(c->d_xbuf);
    if (c->comm) { NcclApi* N = nccl_api(); if (N) N->CommDestroy(c->comm); c->comm = nullptr; }
#endif
    cudaFree(c->d_partials); cudaFree(c->d_done); cudaFreeHost(c->h_out); cudaFree(c->d_q_d2);
    frame_free(c);
    assess_free(c);
    replay_free(c);
    snap_free(c);
    if (c->ev0) cudaEventDestroy(c->ev0);
    if (c->ev1) cudaEventDestroy(c->ev1);
    if (c->evm) cudaEventDestroy(c->evm);
    if (c->own_stream) cudaStreamDestroy(c->own_stream);
    delete h;
    return LIINIT_OK;
}

int liinit_set_stream(liinit_ctx* h, void* cuda_stream) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    CU(cudaStreamSynchronize(c->stream));
    c->stream = cuda_stream ? (cudaStream_t)cuda_stream : c->own_stream;
    return LIINIT_OK;
}

int liinit_get_stream(liinit_ctx* h, void** cuda_stream) {
    if (!h || !cuda_stream) return LIINIT_ERR_INVALID;
    *cuda_stream = (void*)h->c.stream;
    return LIINIT_OK;
}

}  // extern "C"

namespace {
// liinit_map_build and its device twin (dev: xyz is device memory, checked by the caller)
int map_build(Ctx* c, const float* xyz, int stride, int n, bool dev) {
    if (n > c->cfg.max_map_points) return fail(c, LIINIT_ERR_CAPACITY, "n exceeds max_map_points");
    c->map_epoch++;
    // KD_TREE::Build replaces the tree (ikd_Tree.cpp:337-339)
    CU(cudaMemsetAsync(c->d_counters, 0, sizeof(int) * CNT_COUNT, c->stream));
    CU(cudaMemsetAsync(c->M.pool_top, 0, sizeof(unsigned long long), c->stream));
    k_map_clear<<<nblk(c->hash_slots, 256), 256, 0, c->stream>>>(c->M.ent, c->M.aux, c->hash_slots);
    c->launches++;
    if (c->cells) {
        k_sb_clear<<<nblk(c->hash_slots, 256), 256, 0, c->stream>>>(c->M);
        c->launches++;
    }
    // (the retained Nearest_Points are copies: a reuse pass / map_incremental after a map change works on them as in the reference)
    for (long long off = 0; off < n; off += c->stage_pts_cap) {
        int m = (int)((n - off < c->stage_pts_cap) ? (n - off) : c->stage_pts_cap);
        const float4* pts = nullptr;
        int r = stage_batch(c, xyz + (size_t)off * stride, stride, m, dev, &pts);
        if (r) return r;
        r = plain_insert(c, pts, m, nullptr, 0);
        if (r) return r;
        // the staging buffers are reused by the next chunk (the host copy is not stream-ordered against the caller's buffer)
        if (!dev) CU(cudaStreamSynchronize(c->stream));
    }
    int r = fetch_counters(c);
    if (r) return r;
    return check_map_err(c);
}
}  // namespace

extern "C" {

int liinit_map_build(liinit_ctx* h, const float* xyz, int stride, int n) {
    if (!h || (!xyz && n > 0) || n < 0) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    return map_build(c, xyz, stride, n, false);
}

int liinit_map_build_device(liinit_ctx* h, const float* xyz, int stride, int n) {
    if (!h || n < 0) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    int r = device_twin_check(c, stride);
    if (!r && n > 0) r = check_device_ptr(c, xyz, "xyz");
    if (r) return r;
    return map_build(c, xyz, stride, n, true);
}

}  // extern "C"

namespace {
// Slabs only ever grow from the bump allocator and a brick emptied by deletes keeps its slab and its hash slot: a sliding local map
// (Add_Points ahead, Delete_Point_Boxes behind) would run the pool dry although few points are alive. Compaction = flatten the live
// points, clear hash + pool, re-insert them (the Build path): every brick gets one tight slab, empty bricks disappear.
int compact_map(Ctx* c) {
    c->map_epoch++;
    int r = fetch_counters(c);
    if (r) return r;
    const int live = c->h_counters[CNT_LIVE];
    DevBuf<float4> btmp;
    DevBuf<int> bn;
    float4* d_tmp = nullptr;
    int* d_n = nullptr;
    if (live > 0) {
        CU(btmp.alloc((size_t)live));
        CU(bn.alloc(1));
        d_tmp = btmp.p;
        d_n = bn.p;
        CU(cudaMemsetAsync(d_n, 0, sizeof(int), c->stream));
        k_map_flatten4<<<nblk((long long)c->h_counters[CNT_BRICKS] * 32, 256), 256, 0, c->stream>>>(c->M, c->hash_slots, d_tmp, live, d_n);
        c->launches++;
    }
    CU(cudaMemsetAsync(c->d_counters, 0, sizeof(int) * CNT_COUNT, c->stream));
    CU(cudaMemsetAsync(c->M.pool_top, 0, sizeof(unsigned long long), c->stream));
    k_map_clear<<<nblk(c->hash_slots, 256), 256, 0, c->stream>>>(c->M.ent, c->M.aux, c->hash_slots);
    c->launches++;
    if (c->cells) {
        k_sb_clear<<<nblk(c->hash_slots, 256), 256, 0, c->stream>>>(c->M);
        c->launches++;
    }
    r = LIINIT_OK;
    for (long long off = 0; off < live && r == LIINIT_OK; off += c->stage_pts_cap) {
        const int m = (int)((live - off < c->stage_pts_cap) ? (live - off) : c->stage_pts_cap);
        r = plain_insert(c, d_tmp + off, m, nullptr, 0);
    }
    if (r == LIINIT_OK) r = fetch_counters(c);   // (synchronises: the scratch may go)
    else cudaStreamSynchronize(c->stream);
    if (r) return r;
    return check_map_err(c);
}

// Before an update of up to `incoming` points: compact when the allocator is in its last quarter and at least half of what it
// handed out is dead (abandoned slabs, deleted points).
int maybe_compact(Ctx* c, long long incoming) {
    const unsigned long long top = *c->h_pool_top, cap = c->M.pool_cap;
    const long long live = c->h_counters[CNT_LIVE];
    if (top + (unsigned long long)(3 * incoming) + (1ull << 16) > cap - cap / 4 && (unsigned long long)(2 * live) < top) return compact_map(c);
    return LIINIT_OK;
}
}  // namespace

extern "C" {

int liinit_map_compact(liinit_ctx* h) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    return compact_map(c);
}

}  // extern "C"

namespace {
// liinit_map_add_points and its device twin (dev: xyz is device memory, checked by the caller)
int map_add_points(Ctx* c, const float* xyz, int stride, int n, int downsample_on, int* added, bool dev) {
    c->map_epoch++;
    {
        int r = maybe_compact(c, n);
        if (r) return r;
    }
    int total = 0;
    for (long long off = 0; off < n; off += c->stage_pts_cap) {
        int m = (int)((n - off < c->stage_pts_cap) ? (n - off) : c->stage_pts_cap);
        const float4* pts = nullptr;
        int r = stage_batch(c, xyz + (size_t)off * stride, stride, m, dev, &pts);
        if (r) return r;
        r = downsample_on ? downsample_insert(c, pts, m, nullptr, 0) : plain_insert(c, pts, m, nullptr, 0);
        if (r) return r;
        r = fetch_counters(c);
        if (r) return r;
        r = check_map_err(c);
        if (r) return r;
        total += downsample_on ? c->h_counters[CNT_CHANGED] : m;
    }
    if (added) *added = total;
    return LIINIT_OK;
}
}  // namespace

extern "C" {

int liinit_map_add_points(liinit_ctx* h, const float* xyz, int stride, int n, int downsample_on, int* added) {
    if (!h || (!xyz && n > 0) || n < 0) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    return map_add_points(c, xyz, stride, n, downsample_on, added, false);
}

int liinit_map_add_points_device(liinit_ctx* h, const float* xyz, int stride, int n, int downsample_on, int* added) {
    if (!h || n < 0) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    int r = device_twin_check(c, stride);
    if (!r && n > 0) r = check_device_ptr(c, xyz, "xyz");
    if (r) return r;
    return map_add_points(c, xyz, stride, n, downsample_on, added, true);
}

int liinit_map_delete_boxes(liinit_ctx* h, const float* boxes, int nbox, int* deleted) {
    if (!h || (!boxes && nbox > 0) || nbox < 0) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    if (deleted) *deleted = 0;
    if (nbox == 0) return LIINIT_OK;
    c->map_epoch++;
    if ((size_t)nbox * 6 > c->stage_raw_floats) return fail(c, LIINIT_ERR_CAPACITY, "too many boxes");
    CU(cudaMemcpyAsync(c->d_stage_raw, boxes, (size_t)nbox * 6 * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemsetAsync(c->d_vg_misc + 6, 0, sizeof(int), c->stream));
    {   // bricks created so far (the counters are fetched at the end of every map update)
        int r = fetch_counters(c);
        if (r) return r;
    }
    if (c->h_counters[CNT_BRICKS] <= 0) return LIINIT_OK;
    k_map_delete_boxes<<<nblk((long long)c->h_counters[CNT_BRICKS] * 32, 256), 256, 0, c->stream>>>(c->M, c->hash_slots, c->d_stage_raw, nbox,
                                                                                          c->d_vg_misc + 6);
    c->launches++;
    if (c->cells) {
        if (c->cells_refresh_warp) k_cells_refresh_all_warp<<<c->num_sms * 16, 128, 0, c->stream>>>(c->M, c->hash_slots);
        else k_cells_refresh_all<<<nblk(c->hash_slots, 128), 128, 0, c->stream>>>(c->M, c->hash_slots);
        c->launches++;
    }
    CU(cudaGetLastError());
    int cnt = 0;
    CU(cudaMemcpyAsync(&cnt, c->d_vg_misc + 6, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    if (deleted) *deleted = cnt;
    return LIINIT_OK;
}

int liinit_map_validnum(liinit_ctx* h, int* n) {
    if (!h || !n) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    int r = fetch_counters(c);
    if (r) return r;
    *n = c->h_counters[CNT_LIVE];
    return LIINIT_OK;
}

int liinit_map_size(liinit_ctx* h, int* n) { return liinit_map_validnum(h, n); }

int liinit_map_stats(liinit_ctx* h, int* bricks, int* hash_slots, long long* pool_used, long long* pool_cap) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    int r = fetch_counters(c);
    if (r) return r;
    unsigned long long top = 0;
    CU(cudaMemcpyAsync(&top, c->M.pool_top, 8, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    if (bricks) *bricks = c->h_counters[CNT_BRICKS];
    if (hash_slots) *hash_slots = (int)c->hash_slots;
    if (pool_used) *pool_used = (long long)top;
    if (pool_cap) *pool_cap = (long long)c->M.pool_cap;
    return LIINIT_OK;
}

}  // extern "C"

namespace {
// liinit_map_download and its device twin: the live points as packed xyz into xyz [cap*3], their number into *d_n (both device memory)
int map_flatten(Ctx* c, float* xyz, int cap, int* d_n) {
    int r = fetch_counters(c);   // the brick count sizes the launch
    if (r) return r;
    CU(cudaMemsetAsync(d_n, 0, sizeof(int), c->stream));
    if (c->h_counters[CNT_BRICKS] > 0)
        k_map_flatten<<<nblk((long long)c->h_counters[CNT_BRICKS] * 32, 256), 256, 0, c->stream>>>(c->M, c->hash_slots, xyz, cap, d_n);
    c->launches++;
    CU(cudaGetLastError());
    return LIINIT_OK;
}

// The 5-NN of m staged queries for both stand-alone searches: the query kernel of the context's index leaves ids in d_near_ids (the
// search pass's hand-over buffer, free between passes) and distances in d_q_d2, both sized for one staging chunk; k_query_finish then
// writes the outputs (device memory, any may be null).
int query_batch(Ctx* c, const float4* pts, int m, float* out_xyz, float* out_d2, int* out_cnt) {
    if (c->cells) {
        const int gq = nblk(m, LI_CELLS_THREADS);
        if (c->cells_search == 1) k_knn_cells_queries<1><<<gq, LI_CELLS_THREADS, 0, c->stream>>>(c->M, pts, m, c->d_near_ids, c->d_q_d2, c->rho2);
        else if (c->cells_search == 2) k_knn_cells_queries<2><<<gq, LI_CELLS_THREADS, 0, c->stream>>>(c->M, pts, m, c->d_near_ids, c->d_q_d2, c->rho2);
        else k_knn_cells_queries<3><<<gq, LI_CELLS_THREADS, 0, c->stream>>>(c->M, pts, m, c->d_near_ids, c->d_q_d2, c->rho2);
    } else {
        int grid = nblk((long long)m * 8, 256);
        if (grid > c->max_blocks) grid = c->max_blocks;
        k_knn_queries<8><<<grid, 256, 0, c->stream>>>(c->M, pts, m, c->d_near_ids, c->d_q_d2, c->rho2);
    }
    k_query_finish<<<nblk(m, 256), 256, 0, c->stream>>>(c->M.pool, c->d_near_ids, c->d_q_d2, m, out_xyz, out_d2, out_cnt);
    c->launches += 2;
    CU(cudaGetLastError());
    return LIINIT_OK;
}

// liinit_scan_upload and its device twin (dev: body is device memory, checked by the caller)
int scan_upload(Ctx* c, const float* body, int stride, int n, bool dev) {
    if (n > c->cfg.max_scan_points) return fail(c, LIINIT_ERR_CAPACITY, "n exceeds max_scan_points");
    if (stride != 3 && stride != 4 && stride != 12) return fail(c, LIINIT_ERR_INVALID, "stride_floats must be 3, 4 or 12");
    if (stride == 4 && (!dev || aligned16(body))) {
        CU(cudaMemcpyAsync(c->d_body, body, (size_t)n * 16, dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, c->stream));
    } else {
        if (!dev) {   // a host array goes through the strided staging buffer
            const size_t nf = (size_t)n * stride;
            if (nf > c->stage_raw_floats) return fail(c, LIINIT_ERR_CAPACITY, "scan exceeds staging capacity");
            CU(cudaMemcpyAsync(c->d_stage_raw, body, nf * 4, cudaMemcpyHostToDevice, c->stream));
            body = c->d_stage_raw;
        }
        k_repack<<<nblk(n, 256), 256, 0, c->stream>>>(body, stride, n, c->d_body);
        c->launches++;
    }
    c->attached = nullptr;
    c->attached_slot_done = false;
    c->body_attr = false;
    // new scan: no neighbours, nothing selected (Nearest_Points / point_selected_surf start over at iteration 0)
    set_scan(c, n);
    CU(cudaGetLastError());
    return LIINIT_OK;
}

// liinit_raw_upload and its device twin (dev: pts is device memory, checked here after the layout)
int raw_upload(Ctx* c, const float* pts, int stride, int time_index, int n, bool dev) {
    if (stride < 3 || time_index >= stride || (time_index >= 0 && time_index < 3)) return fail(c, LIINIT_ERR_INVALID, "bad stride / time_index");
    if (dev) {
        int r = check_device_ptr(c, pts, "pts");
        if (r) return r;
    }
    if (n > c->stage_pts_cap || (size_t)n * stride > c->stage_raw_floats) return fail(c, LIINIT_ERR_CAPACITY, "raw cloud exceeds staging capacity");
    if (!dev) {
        CU(cudaMemcpyAsync(c->d_stage_raw, pts, (size_t)n * stride * 4, cudaMemcpyHostToDevice, c->stream));
        pts = c->d_stage_raw;
    }
    // the PointType layout (the time in curvature) brings its normals and intensity along; any other layout has none
    c->stage_attr = stride >= 12 && time_index == 9;
    k_repack_t<<<nblk(n, 256), 256, 0, c->stream>>>(pts, stride, time_index, n, c->d_stage_pts, c->stage_attr ? c->d_stage_attr : nullptr);
    c->launches++;
    c->raw_n = n;
    c->stage_seq++;
    CU(cudaGetLastError());
    return LIINIT_OK;
}
}  // namespace

extern "C" {

int liinit_map_download(liinit_ctx* h, float* xyz, int cap, int* n) {
    if (!h || !n || cap < 0) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    DevBuf<float> out;
    DevBuf<int> dn;
    CU(out.alloc((size_t)(cap > 0 ? cap : 1) * 3));
    CU(dn.alloc(1));
    int r = map_flatten(c, out.p, cap, dn.p);
    if (r) return r;
    int cnt = 0;
    CU(cudaMemcpyAsync(&cnt, dn.p, 4, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    const int m = cnt < cap ? cnt : cap;
    if (m > 0 && xyz) {
        CU(cudaMemcpyAsync(xyz, out.p, (size_t)m * 12, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
    }
    *n = cnt;
    return LIINIT_OK;
}

int liinit_map_download_device(liinit_ctx* h, float* xyz, int cap, int* d_n) {
    if (!h || cap < 0) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    int r = device_twin_check(c, 3);
    if (!r) r = check_device_ptr(c, d_n, "d_n");
    if (!r && cap > 0) r = check_device_ptr(c, xyz, "xyz");
    if (r) return r;
    return map_flatten(c, xyz, cap, d_n);
}

int liinit_map_nearest_search(liinit_ctx* h, const float* q, int stride, int n, double max_dist, float* out_xyz, float* out_d2,
                              int* out_cnt) {
    if (!h || !q || n < 0) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    if (max_dist != 5.0) return fail(c, LIINIT_ERR_INVALID, "only max_dist = 5 (laserMapping.cpp:980) is supported");
    CU(cudaSetDevice(c->device));
    // per chunk of the staging capacity: the queries are staged, searched into one device buffer (the wanted outputs of a chunk) and
    // copied back in stream order
    const int chunk = n < c->stage_pts_cap ? n : c->stage_pts_cap;
    const size_t nx = out_xyz ? (size_t)chunk * 15 : 0, nd = out_d2 ? (size_t)chunk * 5 : 0, nc = out_cnt ? (size_t)chunk : 0;
    DevBuf<float> out;
    if (nx + nd + nc > 0) CU(out.alloc(nx + nd + nc));
    float* d_xyz = out_xyz ? out.p : nullptr;
    float* d_d2 = out_d2 ? out.p + nx : nullptr;
    int* d_cnt = out_cnt ? reinterpret_cast<int*>(out.p + nx + nd) : nullptr;
    for (long long off = 0; off < n; off += c->stage_pts_cap) {
        const int m = (int)((n - off < c->stage_pts_cap) ? (n - off) : c->stage_pts_cap);
        int r = stage_points(c, q + (size_t)off * stride, stride, m);
        if (!r) r = query_batch(c, c->d_stage_pts, m, d_xyz, d_d2, d_cnt);
        if (r) return r;
        if (out_xyz) CU(cudaMemcpyAsync(out_xyz + (size_t)off * 15, d_xyz, (size_t)m * 15 * 4, cudaMemcpyDeviceToHost, c->stream));
        if (out_d2) CU(cudaMemcpyAsync(out_d2 + (size_t)off * 5, d_d2, (size_t)m * 5 * 4, cudaMemcpyDeviceToHost, c->stream));
        if (out_cnt) CU(cudaMemcpyAsync(out_cnt + off, d_cnt, (size_t)m * 4, cudaMemcpyDeviceToHost, c->stream));
    }
    CU(cudaStreamSynchronize(c->stream));
    return LIINIT_OK;
}

int liinit_map_nearest_search_device(liinit_ctx* h, const float* q, int stride, int n, double max_dist, float* out_xyz, float* out_d2,
                                     int* out_cnt) {
    if (!h || n < 0) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    if (max_dist != 5.0) return fail(c, LIINIT_ERR_INVALID, "only max_dist = 5 (laserMapping.cpp:980) is supported");
    CU(cudaSetDevice(c->device));
    int r = device_twin_check(c, stride);
    if (!r) r = check_device_ptr(c, q, "q_xyz");
    if (!r && out_xyz) r = check_device_ptr(c, out_xyz, "out_xyz");
    if (!r && out_d2) r = check_device_ptr(c, out_d2, "out_d2");
    if (!r && out_cnt) r = check_device_ptr(c, out_cnt, "out_cnt");
    if (r) return r;
    for (long long off = 0; off < n; off += c->stage_pts_cap) {
        const int m = (int)((n - off < c->stage_pts_cap) ? (n - off) : c->stage_pts_cap);
        const float4* pts = nullptr;
        r = stage_points_device(c, q + (size_t)off * stride, stride, m, &pts);
        if (!r) r = query_batch(c, pts, m, out_xyz ? out_xyz + (size_t)off * 15 : nullptr, out_d2 ? out_d2 + (size_t)off * 5 : nullptr,
                                out_cnt ? out_cnt + off : nullptr);
        if (r) return r;
    }
    return LIINIT_OK;
}

int liinit_scan_upload(liinit_ctx* h, const float* body, int stride, int n) {
    if (!h || !body || n <= 0) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    return scan_upload(c, body, stride, n, false);
}

int liinit_scan_upload_device(liinit_ctx* h, const float* body, int stride, int n) {
    if (!h || n <= 0) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    int r = device_twin_check(c, stride);
    if (!r) r = check_device_ptr(c, body, "body_xyz");
    if (r) return r;
    return scan_upload(c, body, stride, n, true);
}

int liinit_scan_attach_host(liinit_ctx* h, const float* pinned_body, int stride, int n) {
    if (!h || !pinned_body || n <= 0) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    if (n > c->cfg.max_scan_points) return fail(c, LIINIT_ERR_CAPACITY, "n exceeds max_scan_points");
    if (stride != 3 && stride != 4 && stride != 12) return fail(c, LIINIT_ERR_INVALID, "stride_floats must be 3, 4 or 12");
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, pinned_body) != cudaSuccess || at.type != cudaMemoryTypeHost || !at.devicePointer) {
        cudaGetLastError();
        return fail(c, LIINIT_ERR_INVALID, "scan_attach_host needs page-locked, device-mapped host memory (cudaHostAlloc / cudaHostRegister)");
    }
    c->attached = (const float*)at.devicePointer;
    c->attached_stride = stride;
    c->attached_slot_done = false;
    c->body_attr = false;
    set_scan(c, n);   // (N > 1: the search kernel reads this rank's slot in place; the rest is copied when map_incremental / a download needs it)
    return LIINIT_OK;
}

int liinit_raw_upload(liinit_ctx* h, const float* pts, int stride, int time_index, int n) {
    if (!h || !pts || n <= 0) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    return raw_upload(c, pts, stride, time_index, n, false);
}

int liinit_raw_upload_device(liinit_ctx* h, const float* pts, int stride, int time_index, int n) {
    if (!h || n <= 0) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    if (has_comm(c)) return fail(c, LIINIT_ERR_INVALID, "the device-pointer entry points do not take a communicator (liinit_comm_init)");
    return raw_upload(c, pts, stride, time_index, n, true);
}

static int raw_time_range(Ctx* c) {
    const int neg = (int)0xff800000 ^ 0x7fffffff;   // ordered-int image of -inf
    const unsigned long long big = ~0ull;
    CU(cudaMemcpyAsync(c->d_vg_misc + 5, &neg, sizeof(int), cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(c->d_tmin_idx, &big, 8, cudaMemcpyHostToDevice, c->stream));
    k_time_range<<<nblk(c->raw_n, 256), 256, 0, c->stream>>>(c->d_stage_pts, c->raw_n, c->d_tmin_idx, c->d_vg_misc + 5);
    c->launches++;
    return LIINIT_OK;
}

int liinit_raw_undistort_cv(liinit_ctx* h, const double omega[3], const double rot_end[9], const double vel_end[3]) {
    if (!h || !omega || !rot_end || !vel_end) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    if (c->raw_n <= 0) return fail(c, LIINIT_ERR_INVALID, "no raw cloud staged (liinit_raw_upload)");
    int r = raw_time_range(c);
    if (r) return r;
    CvParams P;
    for (int a = 0; a < 3; a++) {
        P.omega[a] = omega[a];
        P.vb[a] = rot_end[a] * vel_end[0] + rot_end[3 + a] * vel_end[1] + rot_end[6 + a] * vel_end[2];   // rot_end^T vel_end
    }
    k_undistort_cv<<<nblk(c->raw_n, 256), 256, 0, c->stream>>>(c->d_stage_pts, c->raw_n, P, c->d_vg_misc + 5, c->d_tmin_idx);
    c->launches++;
    CU(cudaGetLastError());
    return LIINIT_OK;
}

int liinit_raw_undistort_imu(liinit_ctx* h, const double* poses, int npose, const double rot_end[9], const double pos_end[3],
                             const double R_LI[9], const double T_LI[3]) {
    if (!h || !poses || npose < 2 || !rot_end || !pos_end || !R_LI || !T_LI) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    if (c->raw_n <= 0) return fail(c, LIINIT_ERR_INVALID, "no raw cloud staged (liinit_raw_upload)");
    if (npose > LIINIT_MAX_IMU_POSES) return fail(c, LIINIT_ERR_CAPACITY, "IMU pose table too long");
    CU(cudaMemcpyAsync(c->d_poses, poses, (size_t)npose * LI_POSE6D_DOUBLES * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    PoseD S;
    fill_pose(S, rot_end, pos_end, R_LI, T_LI);
    k_undistort_imu<<<nblk(c->raw_n, 256), 256, 0, c->stream>>>(c->d_stage_pts, c->raw_n, c->d_poses, npose, S);
    c->launches++;
    CU(cudaGetLastError());
    return LIINIT_OK;
}

int liinit_frame_cut_livox(liinit_ctx* h, const void* pts, int stride, int n, const liinit_frame_params* p, liinit_subframe* out, int cap,
                           int* n_sub) {
    if (!h || !p || !n_sub || n < 0 || (n > 0 && (!pts || !out))) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    if (stride < 19) return fail(c, LIINIT_ERR_INVALID, "stride_bytes must be at least 19 (CustomPoint)");
    int R = 1;
    int r = frame_check(c, p, n, cap, false, &R);
    if (r) return r;
    *n_sub = 0;
    if (n == 0) return LIINIT_OK;
    r = frame_alloc(c, (size_t)n * stride);
    if (r) return r;
    CU(cudaMemcpyAsync(c->d_fr_in, pts, (size_t)n * stride, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemsetAsync(c->d_fr_tab, 0, offsetof(FrameTable, sub), c->stream));
    const int nb = nblk(n, LI_FR_TILE);
    int* tsum = c->d_fr_tsum;
    int* tsum2 = c->d_fr_tsum + frame_tiles(c);
    k_fr_lvx_valid<<<nb, LI_FR_TILE, 0, c->stream>>>(c->d_fr_in, stride, n, p->N_SCANS, c->d_fr_flag, tsum);
    k_rs_scan<<<1, 1024, 0, c->stream>>>(nb, tsum);
    k_fr_lvx_keep<<<nb, LI_FR_TILE, 0, c->stream>>>(c->d_fr_in, stride, n, p->N_SCANS, p->point_filter_num, p->blind * p->blind, tsum, c->d_fr_flag,
                                                    c->d_fr_dec, c->d_fr_inten, tsum2);
    c->launches += 3;
    CU(cudaGetLastError());
    return frame_finish(c, n, R, p->stamp * 1000, tsum2, out, n_sub);
}

int liinit_frame_cut_pcl2(liinit_ctx* h, const void* data, const liinit_pcl2_layout* lay, int n, const liinit_frame_params* p,
                          liinit_subframe* out, int cap, int* n_sub) {
    if (!h || !p || !lay || !n_sub || n < 0 || (n > 0 && (!data || !out))) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    int R = 1;
    int r = frame_check(c, p, n, cap, true, &R);
    if (r) return r;
    const int t = p->lidar_type;
    const int isz = t == LIINIT_LIDAR_ROBOSENSE ? 1 : 4;
    const int tsz = (t == LIINIT_LIDAR_PANDAR || t == LIINIT_LIDAR_ROBOSENSE) ? 8 : 4;
    const int rsz = t == LIINIT_LIDAR_OUSTER ? 1 : 2;
    const int offs[6] = {lay->off_x, lay->off_y, lay->off_z, lay->off_intensity, lay->off_time, lay->off_ring};
    const int sizes[6] = {4, 4, 4, isz, tsz, rsz};
    if (lay->point_step <= 0) return fail(c, LIINIT_ERR_INVALID, "point_step must be positive");
    for (int f = 0; f < 6; f++)
        if (offs[f] < -1 || (offs[f] >= 0 && offs[f] + sizes[f] > lay->point_step))
            return fail(c, LIINIT_ERR_INVALID, "a field lies outside point_step");
    *n_sub = 0;
    if (n == 0) return LIINIT_OK;
    Pcl2Dev L{lay->point_step, lay->off_x, lay->off_y, lay->off_z, lay->off_intensity, lay->off_time, lay->off_ring, t, 0, 0.0};
    const unsigned char* bytes = static_cast<const unsigned char*>(data);
    if (t == LIINIT_LIDAR_VELO || t == LIINIT_LIDAR_ROBOSENSE) {
        // the rotation model runs when the LAST point's time field is not positive (preprocess.cpp:133,246)
        double last = 0.0;
        if (lay->off_time >= 0) {
            const unsigned char* q = bytes + (size_t)(n - 1) * lay->point_step + lay->off_time;
            if (t == LIINIT_LIDAR_VELO) { float v; memcpy(&v, q, 4); last = v; }
            else memcpy(&last, q, 8);
        }
        L.yaw = !(last > 0);
    }
    if (t == LIINIT_LIDAR_PANDAR && lay->off_time >= 0) memcpy(&L.ts0, bytes + lay->off_time, 8);
    r = frame_alloc(c, (size_t)n * lay->point_step);
    if (r) return r;
    CU(cudaMemcpyAsync(c->d_fr_in, data, (size_t)n * lay->point_step, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemsetAsync(c->d_fr_tab, 0, offsetof(FrameTable, sub), c->stream));
    const int nb = nblk(n, LI_FR_TILE);
    int* tsum = c->d_fr_tsum;
    k_fr_pcl2_decode<<<nb, LI_FR_TILE, 0, c->stream>>>(c->d_fr_in, n, L, p->N_SCANS, p->point_filter_num, p->blind * p->blind, p->stamp,
                                                       c->d_fr_flag, c->d_fr_dec, c->d_fr_inten, c->d_fr_aux, tsum, &c->d_fr_tab->err);
    c->launches++;
    if (L.yaw) {
        // survivors of the blind / NaN test, stably sorted by ring (one 8-bit pass: rings >= 255 are clamped, >= 128 is an error)
        int* ring_first = c->d_fr_ring;
        int* ring_desc = c->d_fr_ring + 256;
        int* n_surv = c->d_fr_ring + 512;
        float* base = reinterpret_cast<float*>(c->d_fr_aux);
        k_rs_scan<<<1, 1024, 0, c->stream>>>(nb, tsum);
        k_fr_compact<<<nb, LI_FR_TILE, 0, c->stream>>>(c->d_fr_flag, n, tsum, c->d_fr_dec, c->d_fr_aux, c->d_fr_keys, c->d_fr_vals, n_surv);
        unsigned* const k[2] = {c->d_fr_keys, c->d_rs_keys};
        unsigned* const v[2] = {c->d_fr_vals, c->d_rs_vals};
        int cur = 0;
        rs_pass(c, k, v, cur, c->d_rs_hist, n, n_surv, 0);   // -> d_rs_keys / d_rs_vals
        k_fr_yaw_first<<<nblk(n, 256), 256, 0, c->stream>>>(c->d_rs_keys, c->d_rs_vals, n_surv, c->d_fr_dec, c->d_fr_yaw, ring_first, ring_desc);
        k_fr_yaw_base<<<nblk(n, 256), 256, 0, c->stream>>>(c->d_rs_keys, n_surv, c->d_fr_yaw, ring_first, base, ring_desc);
        k_fr_yaw_final<<<nblk(n, 256), 256, 0, c->stream>>>(c->d_rs_keys, c->d_rs_vals, n_surv, base, ring_first, ring_desc, p->N_SCANS,
                                                           p->point_filter_num, c->d_fr_dec, c->d_fr_flag, &c->d_fr_tab->err);
        k_fr_yaw_chain<<<1, 256, 0, c->stream>>>(c->d_rs_keys, c->d_rs_vals, n_surv, base, ring_first, &c->d_fr_tab->err, c->d_fr_dec);
        k_fr_tile_count<<<nb, LI_FR_TILE, 0, c->stream>>>(c->d_fr_flag, n, tsum);
        c->launches += 7;
    }
    CU(cudaGetLastError());
    return frame_finish(c, n, R, p->stamp * 1000, tsum, out, n_sub);
}

int liinit_frame_stage(liinit_ctx* h, long long handle) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    int slot = 0;
    const FrameSub* s = frame_lookup(c, handle, &slot);
    if (!s) return fail(c, LIINIT_ERR_INVALID, "unknown sub-frame handle (its message slot has been reused)");
    const size_t o = (size_t)slot * c->stage_pts_cap + (s->lo - 1);
    CU(cudaMemcpyAsync(c->d_stage_pts, c->d_fr_slot_pts + o, (size_t)s->n * sizeof(float4), cudaMemcpyDeviceToDevice, c->stream));
    k_attr_from_inten<<<nblk(s->n, 256), 256, 0, c->stream>>>(c->d_fr_slot_inten + o, s->n, c->d_stage_attr);
    c->launches++;
    CU(cudaGetLastError());
    c->stage_attr = true;
    c->raw_n = s->n;
    c->stage_seq++;
    return LIINIT_OK;
}

int liinit_frame_download(liinit_ctx* h, long long handle, float* pts12, int cap, int* n) {
    if (!h || !n) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    int slot = 0;
    const FrameSub* s = frame_lookup(c, handle, &slot);
    if (!s) return fail(c, LIINIT_ERR_INVALID, "unknown sub-frame handle (its message slot has been reused)");
    *n = s->n;
    if (!pts12) return LIINIT_OK;
    if (cap < s->n) return fail(c, LIINIT_ERR_CAPACITY, "cap_points is smaller than the sub-frame");
    std::vector<float4> P(s->n);
    std::vector<float> I(s->n);
    const size_t o = (size_t)slot * c->stage_pts_cap + (s->lo - 1);
    CU(cudaMemcpyAsync(P.data(), c->d_fr_slot_pts + o, (size_t)s->n * sizeof(float4), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaMemcpyAsync(I.data(), c->d_fr_slot_inten + o, (size_t)s->n * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    for (int i = 0; i < s->n; i++) {
        float* q = pts12 + 12 * (size_t)i;
        q[0] = P[i].x; q[1] = P[i].y; q[2] = P[i].z; q[3] = 1.f;   // PointXYZINormal(): data[3] = 1, normals 0
        q[4] = q[5] = q[6] = q[7] = 0.f;
        q[8] = I[i]; q[9] = P[i].w; q[10] = q[11] = 0.f;
    }
    return LIINIT_OK;
}

int liinit_raw_download(liinit_ctx* h, float* xyz, int cap, int* n) {
    if (!h || !n) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    *n = c->raw_n;
    int m = c->raw_n < cap ? c->raw_n : cap;
    if (m > 0 && xyz) return download_xyz(c, c->d_stage_pts, m, xyz);
    return LIINIT_OK;
}

int liinit_raw_download_world(liinit_ctx* h, const double* R, const double* p, const double* RLI, const double* TLI, float* xyz, int cap,
                              int* n) {
    if (!h || !R || !p || !RLI || !TLI || !n) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    if (c->raw_n <= 0) return fail(c, LIINIT_ERR_INVALID, "no raw cloud staged (liinit_raw_upload)");
    *n = c->raw_n;
    if (!xyz) return LIINIT_OK;
    if (cap < c->raw_n) return fail(c, LIINIT_ERR_CAPACITY, "cap_points is smaller than the staged raw cloud");
    PoseD P;
    fill_pose(P, R, p, RLI, TLI);
    // the strided staging buffer (>= 12 floats per staged point) is free once the cloud has been repacked: it holds the output
    k_raw_to_world<<<nblk(c->raw_n, 256), 256, 0, c->stream>>>(c->d_stage_pts, c->raw_n, P, c->d_stage_raw);
    c->launches++;
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(xyz, c->d_stage_raw, (size_t)c->raw_n * 3 * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return LIINIT_OK;
}

int liinit_raw_downsample(liinit_ctx* h, float leaf_size, int* n_down) {
    if (!h || !(leaf_size > 0.f)) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    const int n = c->raw_n;
    if (n <= 0) return fail(c, LIINIT_ERR_INVALID, "no raw cloud staged (liinit_raw_upload)");
    const int inf_pos = 0x7f800000, inf_neg = (int)0xff800000 ^ 0x7fffffff;   // ordered-int images of +inf / -inf
    const int init[8] = {inf_pos, inf_pos, inf_pos, inf_neg, inf_neg, inf_neg, 0, 0};
    CU(cudaMemcpyAsync(c->d_vg_misc, init, sizeof(init), cudaMemcpyHostToDevice, c->stream));
    VoxTmp V = sized_vox(c, n);
    k_vg_clear<<<nblk((long long)V.mask + 1, 256), 256, 0, c->stream>>>(V, c->d_vg_imin);
    k_vg_minmax<<<nblk(n, 256), 256, 0, c->stream>>>(c->d_stage_pts, n, c->d_vg_misc);
    k_vg_params<<<1, 32, 0, c->stream>>>(c->d_vg_misc, leaf_size, c->d_vg_params);
    k_vg_link<<<nblk(n, 256), 256, 0, c->stream>>>(c->d_stage_pts, n, c->d_vg_params, V, c->d_vg_imin, c->d_vslot_of, c->d_slot_of,
                                                     c->d_vg_misc + 7);
    // one (leaf index, first point) pair per leaf, sorted by leaf index: PCL's output order
    unsigned* const k[2] = {reinterpret_cast<unsigned*>(c->d_flag), c->d_rs_keys};
    unsigned* const v[2] = {reinterpret_cast<unsigned*>(c->d_ins), c->d_rs_vals};
    k_vg_collect<<<nblk((long long)V.mask + 1, 256), 256, 0, c->stream>>>(V, c->d_vg_imin, k[0], v[0], c->d_vg_misc + 6);
    c->launches += 5;
    // the number of leaves is only known on the device: sort with the worst-case tile count, the kernels read the real n
    int cur = 0;
    for (int pass = 0; pass < 4; pass++) rs_pass(c, k, v, cur, c->d_rs_hist, n, c->d_vg_misc + 6, 8 * pass);
    k_vg_centroid_sorted<<<nblk(n, 256), 256, 0, c->stream>>>(c->d_stage_pts, v[cur], c->d_vg_misc + 6, c->d_slot_of, V, c->d_vslot_of, c->d_body,
                                                               c->cfg.max_scan_points, c->d_vg_misc + 7, c->stage_attr ? c->d_stage_attr : nullptr,
                                                               c->d_body_attr);
    c->launches++;
    CU(cudaGetLastError());
    int res[8];
    VgParams P;
    CU(cudaMemcpyAsync(res, c->d_vg_misc, sizeof(res), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaMemcpyAsync(&P, c->d_vg_params, sizeof(P), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    if (P.overflow) return fail(c, LIINIT_ERR_INVALID, "voxel grid: leaf size too small for the cloud extent (index overflow) or no finite point");
    if (res[7] & 1) return fail(c, LIINIT_ERR_CAPACITY, "voxel grid: leaf hash full");
    if (res[7] & 2) return fail(c, LIINIT_ERR_CAPACITY, "voxel grid: more leaves than max_scan_points");
    const int m = res[6];
    if (m <= 0) return fail(c, LIINIT_ERR_INVALID, "voxel grid: no output points");
    set_scan(c, m);
    c->attached = nullptr;
    c->body_attr = c->stage_attr;
    if (n_down) *n_down = m;
    return LIINIT_OK;
}

int liinit_scan_upload_raw(liinit_ctx* h, const float* xyz, int stride, int n, float leaf_size, int* n_down) {
    int r = liinit_raw_upload(h, xyz, stride, -1, n);
    if (r) return r;
    return liinit_raw_downsample(h, leaf_size, n_down);
}

int liinit_scan_download_body(liinit_ctx* h, float* xyz, int cap, int* n) {
    if (!h || !n) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    *n = c->scan_n;
    int m = c->scan_n < cap ? c->scan_n : cap;
    if (m > 0 && xyz) {
        materialize_scan(c);
        return download_xyz(c, c->d_body, m, xyz);
    }
    return LIINIT_OK;
}

int liinit_icp_iterate_device(liinit_ctx* h, const double* R, const double* p, const double* RLI, const double* TLI, int imu_en,
                              int search, double* d_out160) {
    if (!h || !R || !p || !RLI || !TLI || !d_out160) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    return run_pass(c, R, p, RLI, TLI, imu_en, search, d_out160);
}

int liinit_icp_iterate(liinit_ctx* h, const double* R, const double* p, const double* RLI, const double* TLI, int imu_en,
                       int search, double* HtH, double* Htr, int* m, double* res_sq) {
    if (!h || !R || !p || !RLI || !TLI || !HtH || !Htr || !m) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    int r = run_pass(c, R, p, RLI, TLI, imu_en, search, c->h_out_dev);
    if (r) return r;
    CU(cudaStreamSynchronize(c->stream));
    memcpy(HtH, c->h_out, 144 * sizeof(double));
    memcpy(Htr, c->h_out + 144, 12 * sizeof(double));
    if (res_sq) *res_sq = c->h_out[156];
    *m = (int)llround(c->h_out[157]);
    return LIINIT_OK;
}

int liinit_scan_download_state(liinit_ctx* h, float* world_xyz, float* near_xyz, int* near_cnt, unsigned char* selected,
                               float* normvec) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    int n = c->scan_n;
    if (n <= 0) return fail(c, LIINIT_ERR_INVALID, "no scan uploaded");
    {
        int r = init_scan_state(c);
        if (r) return r;
        r = gather_scan_state(c);
        if (r) return r;
    }
    if (world_xyz) {
        int r = download_xyz(c, c->d_world, n, world_xyz);
        if (r) return r;
    }
    CU(cudaStreamSynchronize(c->stream));
    if (near_xyz || near_cnt) {   // Nearest_Points: the device keeps them as point copies (ScanDev::near_xyz, w = 1 found / 0 missing)
        std::vector<float4> nb((size_t)n * 5);
        CU(cudaMemcpy(nb.data(), c->d_near_xyz, (size_t)n * 5 * sizeof(float4), cudaMemcpyDeviceToHost));
        for (int i = 0; i < n; i++) {
            int cnt = 0;
            for (int k = 0; k < 5; k++) {
                const float4& e = nb[(size_t)i * 5 + k];
                const bool ok = e.w != 0.f;
                if (ok) cnt++;
                if (near_xyz) {
                    float* o = near_xyz + 3 * ((size_t)i * 5 + k);
                    o[0] = ok ? e.x : 0.f; o[1] = ok ? e.y : 0.f; o[2] = ok ? e.z : 0.f;
                }
            }
            if (near_cnt) near_cnt[i] = cnt;
        }
    }
    if (selected) CU(cudaMemcpy(selected, c->d_selected, (size_t)n, cudaMemcpyDeviceToHost));
    if (normvec) CU(cudaMemcpy(normvec, c->d_normvec, (size_t)n * 16, cudaMemcpyDeviceToHost));
    return LIINIT_OK;
}

int liinit_scan_download_effect(liinit_ctx* h, float* ori_xyz, float* normvec, int cap, int* m) {
    if (!h || !m) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    int n = c->scan_n;
    if (n <= 0) return fail(c, LIINIT_ERR_INVALID, "no scan uploaded");
    materialize_scan(c);
    {
        int r = init_scan_state(c);
        if (r) return r;
        r = gather_scan_state(c);
        if (r) return r;
    }
    CU(cudaStreamSynchronize(c->stream));
    std::vector<unsigned char> sel(n);
    std::vector<float4> nv(n), body(n);
    CU(cudaMemcpy(sel.data(), c->d_selected, (size_t)n, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(nv.data(), c->d_normvec, (size_t)n * 16, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(body.data(), c->d_body, (size_t)n * 16, cudaMemcpyDeviceToHost));
    int k = 0;
    for (int i = 0; i < n; i++) {   // order-preserving compaction (laserMapping.cpp:1013-1020)
        if (!sel[i]) continue;
        if (k < cap) {
            if (ori_xyz) {
                ori_xyz[3 * (size_t)k] = body[i].x; ori_xyz[3 * (size_t)k + 1] = body[i].y; ori_xyz[3 * (size_t)k + 2] = body[i].z;
            }
            if (normvec) memcpy(normvec + 4 * (size_t)k, &nv[i], 16);
        }
        k++;
    }
    *m = k;
    return LIINIT_OK;
}

}  // extern "C"

namespace {
// liinit_cloud_download and its device twin. dev: the records are built in rec12 (device memory) itself, d_n (device, may be null)
// receives the count; n (host) may then be null, and an EFFECT count is only brought to the host when n asks for it or cap_points
// does not cover the whole resident scan.
int cloud_download(Ctx* c, int which, const double* R, const double* p, const double* RLI, const double* TLI, float* rec12, int cap, int* n,
                   int* d_n, bool dev) {
    if (which < LIINIT_CLOUD_REGISTERED || which > LIINIT_CLOUD_EFFECT) return fail(c, LIINIT_ERR_INVALID, "unknown cloud");
    if (which != LIINIT_CLOUD_BODY && (!R || !p || !RLI || !TLI)) return fail(c, LIINIT_ERR_INVALID, "a world-frame cloud needs the pose");
    const bool raw = which == LIINIT_CLOUD_REGISTERED || which == LIINIT_CLOUD_BODY;
    if (raw && c->raw_n <= 0) return fail(c, LIINIT_ERR_INVALID, "no raw cloud staged (liinit_raw_upload / liinit_frame_stage)");
    if (!raw && c->scan_n <= 0) return fail(c, LIINIT_ERR_INVALID, "no scan resident");
    if (which == LIINIT_CLOUD_EFFECT && !c->have_neighbors) return fail(c, LIINIT_ERR_INVALID, "no ICP pass on the resident scan yet");
    PoseD P;
    if (which != LIINIT_CLOUD_BODY) fill_pose(P, R, p, RLI, TLI);
    // host twin: the records are built in the strided staging buffer (12 floats per point of the staging capacity), free once a cloud
    // is repacked
    float* out = dev ? rec12 : c->d_stage_raw;
    const float4* battr = c->body_attr ? c->d_body_attr : nullptr;
    int m = 0;   // -1: an EFFECT count left on the device (at most scan_n <= cap)
    if (raw) {
        m = c->raw_n;
    } else if (which == LIINIT_CLOUD_REGISTERED_DOWN) {
        m = c->scan_n;
    } else {
        // laserCloudOri: the points the last pass selected, over the whole frame (N > 1: after the all-gather of the flags)
        int r = init_scan_state(c);
        if (r) return r;
        r = gather_scan_state(c);
        if (r) return r;
        const int nb = nblk(c->scan_n, LI_FR_TILE);
        k_eff_count<<<nb, LI_FR_TILE, 0, c->stream>>>(c->d_selected, c->scan_n, c->d_vg_block);
        k_rs_scan<<<1, 1024, 0, c->stream>>>(nb + 1, c->d_vg_block);
        c->launches += 2;
        CU(cudaGetLastError());
        if (d_n) CU(cudaMemcpyAsync(d_n, c->d_vg_block + nb, sizeof(int), cudaMemcpyDeviceToDevice, c->stream));
        if (n || (rec12 && cap < c->scan_n)) {
            CU(cudaMemcpyAsync(&m, c->d_vg_block + nb, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
            CU(cudaStreamSynchronize(c->stream));
        } else {
            m = -1;
        }
    }
    if (n) *n = m;
    if (rec12 && cap < m) return fail(c, LIINIT_ERR_CAPACITY, "cap_points is smaller than the cloud");
    if (d_n && which != LIINIT_CLOUD_EFFECT) {
        k_store_int<<<1, 32, 0, c->stream>>>(d_n, m);
        c->launches++;
    }
    if (!rec12 || m == 0) return LIINIT_OK;
    if (!raw) materialize_scan(c);   // (an attached host scan: the whole frame into d_body)
    const float4* sattr = c->stage_attr ? c->d_stage_attr : nullptr;
    switch (which) {
        case LIINIT_CLOUD_REGISTERED: k_cloud_world<<<nblk(m, 256), 256, 0, c->stream>>>(c->d_stage_pts, sattr, m, P, out); break;
        case LIINIT_CLOUD_BODY: k_cloud_body<<<nblk(m, 256), 256, 0, c->stream>>>(c->d_stage_pts, sattr, m, out); break;
        case LIINIT_CLOUD_REGISTERED_DOWN: k_cloud_world<<<nblk(m, 256), 256, 0, c->stream>>>(c->d_body, battr, m, P, out); break;
        default: k_eff_emit<<<nblk(c->scan_n, LI_FR_TILE), LI_FR_TILE, 0, c->stream>>>(c->d_selected, c->scan_n, c->d_vg_block, c->d_body, battr, P, out); break;
    }
    c->launches++;
    CU(cudaGetLastError());
    if (dev) return LIINIT_OK;
    CU(cudaMemcpyAsync(rec12, out, (size_t)m * 12 * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return LIINIT_OK;
}
}  // namespace

extern "C" {

int liinit_cloud_download(liinit_ctx* h, int which, const double* R, const double* p, const double* RLI, const double* TLI, float* rec12,
                          int cap, int* n) {
    if (!h || !n) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    return cloud_download(c, which, R, p, RLI, TLI, rec12, cap, n, nullptr, false);
}

int liinit_cloud_download_device(liinit_ctx* h, int which, const double* R, const double* p, const double* RLI, const double* TLI, float* rec12,
                                 int cap, int* n, int* d_n) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    int r = device_twin_check(c, 12);
    if (!r && !n && !d_n) r = fail(c, LIINIT_ERR_INVALID, "neither n nor d_n is given");
    if (!r && d_n) r = check_device_ptr(c, d_n, "d_n");
    if (!r && rec12) r = check_device_ptr(c, rec12, "rec12");
    if (!r && rec12 && !aligned16(rec12)) r = fail(c, LIINIT_ERR_INVALID, "rec12 must be 16-byte aligned");
    if (r) return r;
    return cloud_download(c, which, R, p, RLI, TLI, rec12, cap, n, d_n, true);
}

int liinit_map_incremental(liinit_ctx* h, const double* R, const double* p, const double* RLI, const double* TLI, double ds,
                           int flg_EKF_inited, int* n_add, int* n_nod) {
    if (!h || !R || !p || !RLI || !TLI) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    int n = c->scan_n;
    if (n <= 0) return fail(c, LIINIT_ERR_INVALID, "no scan uploaded");
    materialize_scan(c);
    {
        int r = init_scan_state(c);   // no search pass on this scan yet: every point has "no neighbours" (-> PointToAdd)
        if (r) return r;
        // N > 1: the Nearest_Points of the other ranks' shards; then every rank applies the WHOLE frame's update to its replica
        r = gather_scan_state(c);
        if (r) return r;
    }
    c->map_epoch++;
    {
        int r = maybe_compact(c, n);
        if (r) return r;
    }
    PoseD P;
    fill_pose(P, R, p, RLI, TLI);
    static const int zeros[2] = {0, 0};
    CU(cudaMemcpyAsync(c->d_counters + CNT_NADD, zeros, 2 * sizeof(int), cudaMemcpyHostToDevice, c->stream));
    k_incr_classify<<<nblk(n, 256), 256, 0, c->stream>>>(c->M, P, c->d_body, n, c->d_near_xyz, ds, flg_EKF_inited, c->d_world,
                                                        c->d_flag);
    c->launches++;
    CU(cudaGetLastError());
    // Add_Points(PointToAdd, true) then Add_Points(PointNoNeedDownsample, false) (laserMapping.cpp:556-557).
    // d_world (float4) is the point source; it stays untouched by the inserts.
    int r = downsample_insert(c, c->d_world, n, c->d_flag, 1);
    if (r) return r;
    r = plain_insert(c, c->d_world, n, c->d_flag, 2);
    if (r) return r;
    r = fetch_counters(c);
    if (r) return r;
    if (n_add) *n_add = c->h_counters[CNT_NADD];
    if (n_nod) *n_nod = c->h_counters[CNT_NNOD];
    return check_map_err(c);
}

int liinit_last_pass_timing(liinit_ctx* h, float* kernel_ms, int* launches) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    CU(cudaEventSynchronize(c->ev1));
    float ms = 0.f;
    CU(cudaEventElapsedTime(&ms, c->ev0, c->ev1));
    c->last_ms = ms;
    if (kernel_ms) *kernel_ms = ms;
    if (launches) *launches = c->last_launches;
    return LIINIT_OK;
}

int liinit_last_pass_kernel_times(liinit_ctx* h, float* knn_ms, float* plane_ms) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    CU(cudaEventSynchronize(c->ev1));
    float a = 0.f, b = 0.f;
    if (c->last_was_search) {
        CU(cudaEventElapsedTime(&a, c->ev0, c->evm));
        CU(cudaEventElapsedTime(&b, c->evm, c->ev1));
    } else {
        CU(cudaEventElapsedTime(&b, c->ev0, c->ev1));
    }
    if (knn_ms) *knn_ms = a;
    if (plane_ms) *plane_ms = b;
    return LIINIT_OK;
}

int liinit_debug_esti_plane(liinit_ctx* h, const float* nb_xyz, int n, double* pabcd, unsigned char* valid) {
    if (!h || !nb_xyz || !pabcd || !valid || n < 0) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    if (n == 0) return LIINIT_OK;
    float* d_in = nullptr;
    double* d_out = nullptr;
    unsigned char* d_ok = nullptr;
    int rc = LIINIT_OK;
    if (cudaMalloc(&d_in, (size_t)n * 15 * 4) != cudaSuccess || cudaMalloc(&d_out, (size_t)n * 32) != cudaSuccess || cudaMalloc(&d_ok, (size_t)n) != cudaSuccess) {
        rc = fail(c, LIINIT_ERR_CUDA, "cudaMalloc (debug_esti_plane)");
    } else {
        cudaMemcpyAsync(d_in, nb_xyz, (size_t)n * 15 * 4, cudaMemcpyHostToDevice, c->stream);
        k_debug_esti_plane<<<nblk(n, 128), 128, 0, c->stream>>>(d_in, n, d_out, d_ok);
        c->launches++;
        cudaMemcpyAsync(pabcd, d_out, (size_t)n * 32, cudaMemcpyDeviceToHost, c->stream);
        cudaMemcpyAsync(valid, d_ok, (size_t)n, cudaMemcpyDeviceToHost, c->stream);
        cudaError_t e = cudaStreamSynchronize(c->stream);
        if (e == cudaSuccess) e = cudaGetLastError();
        if (e != cudaSuccess) rc = fail(c, LIINIT_ERR_CUDA, std::string("debug_esti_plane: ") + cudaGetErrorString(e));
    }
    cudaFree(d_in); cudaFree(d_out); cudaFree(d_ok);
    return rc;
}

// ---- multi-GPU (SURVEY.md section 8e) -----------------------------------------------------------------------
int liinit_comm_unique_id(void* id128) {
    if (!id128) return LIINIT_ERR_INVALID;
#ifdef LI_SIMT_EMUL
    return LIINIT_ERR_INVALID;
#else
    NcclApi* N = nccl_api();
    if (!N) {
        g_create_error = "NCCL is not available (dlopen libnccl.so.2 failed)";
        return LIINIT_ERR_CUDA;
    }
    static_assert(sizeof(ncclUniqueId) == LIINIT_COMM_ID_BYTES, "ncclUniqueId size");
    ncclUniqueId id;
    ncclResult_t nr = N->GetUniqueId(&id);
    if (nr != ncclSuccess) {
        g_create_error = std::string("ncclGetUniqueId: ") + N->GetErrorString(nr);
        return LIINIT_ERR_CUDA;
    }
    memcpy(id128, &id, sizeof(id));
    return LIINIT_OK;
#endif
}

int liinit_comm_init(liinit_ctx* h, const void* id128, int nranks, int rank) {
    if (!h || !id128 || nranks < 1 || nranks > 64 || rank < 0 || rank >= nranks) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
#ifdef LI_SIMT_EMUL
    return fail(c, LIINIT_ERR_INVALID, "no communicator in the CPU checker");
#else
    CU(cudaSetDevice(c->device));
    if (c->comm) return fail(c, LIINIT_ERR_INVALID, "communicator already attached");
    NcclApi* N = nccl_api();
    if (!N) return fail(c, LIINIT_ERR_CUDA, "NCCL is not available (dlopen libnccl.so.2 failed)");
    CU(cudaStreamSynchronize(c->stream));
    ncclUniqueId id;
    memcpy(&id, id128, sizeof(id));
    ncclResult_t nr = N->CommInitRank(&c->comm, nranks, id, rank);
    if (nr != ncclSuccess) {
        c->comm = nullptr;
        return fail(c, LIINIT_ERR_CUDA, std::string("ncclCommInitRank: ") + N->GetErrorString(nr));
    }
    c->nranks = nranks;
    c->rank = rank;
    if (c->scan_n > 0) set_scan(c, c->scan_n);   // re-cut a frame that is already resident
    // ---- peer-memory exchange (one process per GPU on one NVLink node): every rank's buffer mapped into every process through CUDA IPC.
    // If any rank cannot set it up (same process, no peer access, LIINIT_COMM_MODE=nccl), ALL ranks stay on ncclAllReduce.
    c->comm_p2p = false;
    if (nranks > 1) {
        const char* mode = getenv("LIINIT_COMM_MODE");
        int ok = !(mode && !strcmp(mode, "nccl")) ? 1 : 0;
        const size_t blk_bytes = (size_t)2 * nranks * 160 * sizeof(double), flag_bytes = (size_t)2 * nranks * sizeof(unsigned);
        cudaIpcMemHandle_t mine;
        memset(&mine, 0, sizeof(mine));
        if (ok && (cudaMalloc(&c->d_xbuf, blk_bytes + flag_bytes) != cudaSuccess || cudaMemset(c->d_xbuf, 0, blk_bytes + flag_bytes) != cudaSuccess ||
                   cudaIpcGetMemHandle(&mine, c->d_xbuf) != cudaSuccess)) {
            ok = 0;
            cudaGetLastError();
        }
        // all-gather of the 64-byte handles (+ a 4-byte "fine so far" word) through the communicator that now exists
        const size_t rec = sizeof(cudaIpcMemHandle_t) + 8;
        DevBuf<unsigned char> dh;
        std::vector<unsigned char> hh(rec * nranks, 0);
        if (dh.alloc(rec * nranks) != cudaSuccess) return fail(c, LIINIT_ERR_CUDA, "cudaMalloc (comm handles)");
        memcpy(hh.data() + rec * rank, &mine, sizeof(mine));
        memcpy(hh.data() + rec * rank + sizeof(mine), &ok, sizeof(int));
        CU(cudaMemcpy(dh.p + rec * rank, hh.data() + rec * rank, rec, cudaMemcpyHostToDevice));
        nr = N->AllGather(dh.p + rec * rank, dh.p, rec, ncclChar, c->comm, c->stream);
        if (nr != ncclSuccess) return fail(c, LIINIT_ERR_CUDA, std::string("ncclAllGather (comm handles): ") + N->GetErrorString(nr));
        CU(cudaStreamSynchronize(c->stream));
        CU(cudaMemcpy(hh.data(), dh.p, rec * nranks, cudaMemcpyDeviceToHost));
        for (int r = 0; r < nranks; r++) {
            int okr = 0;
            memcpy(&okr, hh.data() + rec * r + sizeof(mine), sizeof(int));
            ok = ok && okr;
        }
        XchgTable T;
        memset(&T, 0, sizeof(T));
        if (ok) {
            for (int r = 0; r < nranks && ok; r++) {
                void* base = c->d_xbuf;
                if (r != rank) {
                    cudaIpcMemHandle_t hr;
                    memcpy(&hr, hh.data() + rec * r, sizeof(hr));
                    if (cudaIpcOpenMemHandle(&base, hr, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
                        ok = 0;
                        cudaGetLastError();
                        break;
                    }
                    c->peer_map[r] = base;
                }
                T.blocks[r] = (double*)base;
                T.flags[r] = (unsigned*)((unsigned char*)base + blk_bytes);
            }
        }
        // second agreement: did every rank open every handle? (sum of the failures over the ranks)
        {
            DevBuf<double> dv;
            if (dv.alloc(1) != cudaSuccess) return fail(c, LIINIT_ERR_CUDA, "cudaMalloc (comm agreement)");
            double bad = ok ? 0.0 : 1.0;
            CU(cudaMemcpy(dv.p, &bad, sizeof(double), cudaMemcpyHostToDevice));
            nr = N->AllReduce(dv.p, dv.p, 1, ncclDouble, ncclSum, c->comm, c->stream);
            if (nr != ncclSuccess) return fail(c, LIINIT_ERR_CUDA, std::string("ncclAllReduce (comm agreement): ") + N->GetErrorString(nr));
            CU(cudaStreamSynchronize(c->stream));
            CU(cudaMemcpy(&bad, dv.p, sizeof(double), cudaMemcpyDeviceToHost));
            ok = bad == 0.0;
        }
        if (ok) {
            T.local = c->d_acc;
            T.nranks = nranks;
            T.rank = rank;
            CU(cudaMalloc(&c->d_xtab, sizeof(XchgTable)));
            CU(cudaMemcpy(c->d_xtab, &T, sizeof(T), cudaMemcpyHostToDevice));
            c->comm_p2p = true;
            c->xseq = 0;
        }
    }
    return LIINIT_OK;
#endif
}

int liinit_comm_last_local(liinit_ctx* h, double* out160) {
    if (!h || !out160) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    if (c->nranks <= 1) return fail(c, LIINIT_ERR_INVALID, "no communicator attached");
    CU(cudaSetDevice(c->device));
    CU(cudaStreamSynchronize(c->stream));
    CU(cudaMemcpy(out160, c->d_acc, 160 * sizeof(double), cudaMemcpyDeviceToHost));
    return LIINIT_OK;
}

int liinit_comm_mode(liinit_ctx* h, int* peer_memory) {
    if (!h || !peer_memory) return LIINIT_ERR_INVALID;
    *peer_memory = (h->c.nranks > 1 && h->c.comm_p2p) ? 1 : 0;
    return LIINIT_OK;
}

int liinit_comm_info(liinit_ctx* h, int* nranks, int* rank, int* shard_lo, int* shard_n) {
    if (!h) return LIINIT_ERR_INVALID;
    if (nranks) *nranks = h->c.nranks;
    if (rank) *rank = h->c.rank;
    if (shard_lo) *shard_lo = h->c.shard_lo;
    if (shard_n) *shard_n = h->c.S.n;
    return LIINIT_OK;
}

int liinit_set_reseed(liinit_ctx* h, int enabled) {
    if (!h) return LIINIT_ERR_INVALID;
    h->c.reseed = enabled != 0;
    return LIINIT_OK;
}

int liinit_knn_index(liinit_ctx* h, int* knn_index) {
    if (!h || !knn_index) return LIINIT_ERR_INVALID;
    *knn_index = h->c.cells ? LIINIT_KNN_CELLS : LIINIT_KNN_BRICKS;
    return LIINIT_OK;
}

int liinit_launch_count(liinit_ctx* h, long long* launches) {
    if (!h || !launches) return LIINIT_ERR_INVALID;
    *launches = h->c.launches;
    return LIINIT_OK;
}

}  // extern "C"

// ---- map assessment (assess_kernels.cuh, DESIGN.md section 4d) ----
namespace {

int assess_check(Ctx* c) {
    if (has_comm(c)) return fail(c, LIINIT_ERR_INVALID, "the map assessment does not take a communicator (liinit_comm_init)");
    if (c->A.cap == 0) return fail(c, LIINIT_ERR_INVALID, "no assessment store (liinit_assess_reserve)");
    return LIINIT_OK;
}

// the checks liinit_assess_evaluate and liinit_assess_cloud share; a cloud takes every stored point as a query (stride 0 or 1)
int assess_check_params(Ctx* c, const liinit_assess_params* prm, const double* R_LI, const double* T_LI, bool cloud) {
    const double r = prm->radius;
    if (!std::isfinite(r) || !(r > 0.0)) return fail(c, LIINIT_ERR_INVALID, "radius must be positive and finite");
    if (prm->min_neighbors < 4) return fail(c, LIINIT_ERR_INVALID, "min_neighbors must be at least 4");
    if (!cloud && prm->query_stride < 0) return fail(c, LIINIT_ERR_INVALID, "query_stride must be >= 0 (0: automatic)");
    if (cloud && prm->query_stride != 0 && prm->query_stride != 1)
        return fail(c, LIINIT_ERR_INVALID, "a cloud takes every stored point as a query: query_stride must be 0 or 1");
    if (!prm->as_run && (!R_LI || !T_LI)) return fail(c, LIINIT_ERR_INVALID, "a candidate extrinsic needs R_LI and T_LI (or as_run)");
    if (!prm->as_run)
        for (int k = 0; k < 12; k++)
            if (!std::isfinite(k < 9 ? R_LI[k] : T_LI[k - 9])) return fail(c, LIINIT_ERR_INVALID, "R_LI / T_LI must be finite");
    return LIINIT_OK;
}

// k_as_place into A.world (lag: the timed placement, k_at_scan_end + k_at_place, at lag shift *lag), then the grid of cubic cells of
// edge `edge` over the placed bounding box (one synchronisation); leaf: the cells are the leaves of a cloud
int assess_place(Ctx* c, int as_run, const PoseD& cand, double edge, bool leaf, AsGrid& G, const double* lag = nullptr) {
    Ctx::Assess& A = c->A;
    const int n = (int)A.n;
    int box[8] = {0x7fffffff, 0x7fffffff, 0x7fffffff, -0x7fffffff - 1, -0x7fffffff - 1, -0x7fffffff - 1, 0, 0};
    CU(cudaMemcpyAsync(A.box, box, sizeof(box), cudaMemcpyHostToDevice, c->stream));
    if (lag) {
        k_at_scan_end<<<nblk(A.scans, 128), 128, 0, c->stream>>>(A.at, A.pool, A.scans, *lag, as_run, cand, A.at_end);
        k_at_place<<<nblk(n, 256), 256, 0, c->stream>>>(A.pts, A.raw, A.poses, A.at, A.at_end, A.pool, n, *lag, as_run, cand, edge, A.world, A.box);
        c->launches += 2;
    } else {
        k_as_place<<<nblk(n, 256), 256, 0, c->stream>>>(A.pts, A.poses, n, as_run, cand, edge, A.world, A.box);
        c->launches++;
    }
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(box, A.box, sizeof(box), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    if (box[6])
        return fail(c, LIINIT_ERR_CAPACITY, std::string("a placed point is not finite or lies 2^30 ") + (leaf ? "leaves" : "cells") + " or more from the origin");
    G.edge = edge;
    for (int a = 0; a < 3; a++) {
        G.lo[a] = box[a];
        G.ext[a] = (long long)box[3 + a] - box[a] + 1;
    }
    if ((double)G.ext[0] * (double)G.ext[1] * (double)G.ext[2] > 9.0e18)
        return fail(c, LIINIT_ERR_CAPACITY, leaf ? "the placed cloud spans more leaves than a 63-bit leaf key holds"
                                                 : "the placed cloud spans more cells than a 63-bit cell key holds");
    return LIINIT_OK;
}

// keys of A.world on the grid G (A.key) and the stable radix sort of the identity permutation by them: the sorted stored indices end in
// A.v[cur]
int assess_sort(Ctx* c, const AsGrid& G, int& cur) {
    Ctx::Assess& A = c->A;
    const int n = (int)A.n;
    const unsigned long long cells = (unsigned long long)G.ext[0] * (unsigned long long)G.ext[1] * (unsigned long long)G.ext[2];
    int bits = 0;
    while (bits < 64 && ((cells - 1) >> bits)) bits++;
    k_as_key<<<nblk(n, 256), 256, 0, c->stream>>>(A.world, n, G, A.key, A.k[0], A.v[0]);
    c->launches++;
    CU(cudaGetLastError());
    // stable sort by cell key: the low word's digits, then (keys wider than 32 bits) the high word's; only the digits the box needs
    cur = 0;
    for (int sh = 0; sh < bits && sh < 32; sh += 8) rs_pass(c, A.k, A.v, cur, A.hist, n, nullptr, sh);
    if (bits > 32) {
        k_rs_gather_hi<<<nblk(n, 256), 256, 0, c->stream>>>(A.key, A.v[cur], n, A.k[cur]);
        c->launches++;
        for (int sh = 0; sh < bits - 32; sh += 8) rs_pass(c, A.k, A.v, cur, A.hist, n, nullptr, sh);
    }
    CU(cudaGetLastError());
    return LIINIT_OK;
}

// the candidate's extrinsic (unused with as_run)
PoseD assess_candidate(const liinit_assess_params* prm, const double* R_LI, const double* T_LI) {
    PoseD cand{};
    if (!prm->as_run) {
        memcpy(cand.RLI, R_LI, 72);
        memcpy(cand.TLI, T_LI, 24);
    }
    return cand;
}

// the cell edge of a radius: r (1 + 2^-20), see li_as_cell
double assess_edge(double r) { return r * (1.0 + ldexp(1.0, -20)); }

// lag: a timed evaluation at that lag shift (assess_place)
int assess_evaluate(Ctx* c, const liinit_assess_params* prm, const double* R_LI, const double* T_LI, liinit_assess_result* out,
                    const double* lag = nullptr) {
    Ctx::Assess& A = c->A;
    const double r = prm->radius;
    int rc = assess_check_params(c, prm, R_LI, T_LI, false);
    if (rc) return rc;
    if (A.n == 0) return fail(c, LIINIT_ERR_INVALID, "the assessment store is empty (liinit_assess_append)");
    const int n = (int)A.n;
    const long long s = prm->query_stride > 0 ? prm->query_stride : (A.n + LIINIT_ASSESS_MAX_QUERIES - 1) / LIINIT_ASSESS_MAX_QUERIES;
    const long long nq = (A.n + s - 1) / s;
    if (nq > LIINIT_ASSESS_MAX_QUERIES)
        return fail(c, LIINIT_ERR_CAPACITY, "query_stride gives " + std::to_string(nq) + " queries, more than LIINIT_ASSESS_MAX_QUERIES");
    AsGrid G;
    rc = assess_place(c, prm->as_run ? 1 : 0, assess_candidate(prm, R_LI, T_LI), assess_edge(r), false, G, lag);
    if (rc) return rc;
    int cur;
    rc = assess_sort(c, G, cur);
    if (rc) return rc;
    k_as_gather<<<nblk(n, 256), 256, 0, c->stream>>>(A.world, A.key, A.v[cur], n, A.sorted, A.skey);
    c->launches++;
    const int nb = nblk(n, LI_FR_TILE);
    const int qs = (int)s;
    k_as_mark<<<nb, LI_FR_TILE, 0, c->stream>>>(A.skey, A.sorted, n, qs, 0, n, A.tc, A.tq);
    k_rs_scan<<<1, 1024, 0, c->stream>>>(nb + 1, A.tc);
    k_rs_scan<<<1, 1024, 0, c->stream>>>(nb + 1, A.tq);
    k_as_index<<<nb, LI_FR_TILE, 0, c->stream>>>(A.skey, A.sorted, n, qs, 0, n, A.tc, A.tq, A.cell_start, A.cell_key, A.cell_q0, A.qlist);
    // (there are at most n cells: nb blocks cover them)
    k_as_task_count<<<nb, LI_FR_TILE, 0, c->stream>>>(A.cell_q0, A.tc + nb, A.tt);
    k_rs_scan<<<1, 1024, 0, c->stream>>>(nb + 1, A.tt);
    k_as_task_emit<<<nb, LI_FR_TILE, 0, c->stream>>>(A.cell_q0, A.tc + nb, A.tt, A.tasks);
    c->launches += 8;
    CU(cudaGetLastError());
    CU(cudaMemsetAsync(A.ticket, 0, sizeof(unsigned), c->stream));
    k_as_moments<<<c->num_sms * 8, LI_AS_BLOCK, 0, c->stream>>>(A.sorted, A.cell_start, A.cell_key, A.tc + nb, A.qlist, A.tasks, A.tt + nb, A.ticket,
                                                                G, r * r, qs, prm->min_neighbors, A.qn, A.qh, A.qv);
    k_as_reduce<<<1, 1024, 0, c->stream>>>(A.qn, A.qh, A.qv, (int)nq, prm->min_neighbors, A.tot);
    c->launches += 2;
    CU(cudaGetLastError());
    AsTotals T;
    CU(cudaMemcpyAsync(&T, A.tot, sizeof(T), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    A.last_q = nq;
    A.last_n = A.n;
    out->points = A.n;
    out->queries = nq;
    out->stride = qs;
    out->scans = A.scans;
    out->valid = T.valid;
    out->sparse = T.sparse;
    out->degenerate = T.degenerate;
    out->mme = T.valid ? T.sum_h / (double)T.valid : NAN;
    out->mpv = T.valid ? T.sum_v / (double)T.valid : NAN;
    return LIINIT_OK;
}

// stored points per moments batch of a cloud: the per-query buffers liinit_assess_reserve sizes for LIINIT_ASSESS_MAX_QUERIES queries
// hold one batch (a smaller value only splits the work more finely; the CPU tests build one)
#ifndef LI_AS_CLOUD_BATCH
#define LI_AS_CLOUD_BATCH LIINIT_ASSESS_MAX_QUERIES
#endif
static_assert(LI_AS_CLOUD_BATCH > 0 && LI_AS_CLOUD_BATCH <= LIINIT_ASSESS_MAX_QUERIES, "a cloud batch must fit the per-query buffers");

// leaves of A.world on the grid L: the stored indices in leaf order in A.v[cur] (stored order inside a leaf), leaf c at sorted
// positions A.cell_start[c] .. A.cell_start[c + 1]; *leaves = their number (one synchronisation)
int assess_leaf_table(Ctx* c, const AsGrid& L, int& cur, long long& leaves) {
    Ctx::Assess& A = c->A;
    const int n = (int)A.n;
    int rc = assess_sort(c, L, cur);
    if (rc) return rc;
    const int nb = nblk(n, LI_FR_TILE);
    k_ac_leaf_mark<<<nb, LI_FR_TILE, 0, c->stream>>>(A.key, A.v[cur], n, A.tc);
    k_rs_scan<<<1, 1024, 0, c->stream>>>(nb + 1, A.tc);
    k_ac_leaf_index<<<nb, LI_FR_TILE, 0, c->stream>>>(A.key, A.v[cur], n, A.tc, A.cell_start);
    c->launches += 3;
    CU(cudaGetLastError());
    int m = 0;
    CU(cudaMemcpyAsync(&m, A.tc + nb, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    leaves = m;
    return LIINIT_OK;
}

int assess_cloud(Ctx* c, const liinit_assess_params* prm, const double* R_LI, const double* T_LI, double leaf, float* rec8, long long cap,
                 long long* n_out, liinit_assess_result* out) {
    Ctx::Assess& A = c->A;
    int rc = assess_check_params(c, prm, R_LI, T_LI, true);
    if (rc) return rc;
    if (!std::isfinite(leaf) || leaf < 0.0) return fail(c, LIINIT_ERR_INVALID, "leaf must be >= 0 and finite (0: one record per stored point)");
    if (A.n == 0) return fail(c, LIINIT_ERR_INVALID, "the assessment store is empty (liinit_assess_append)");
    const int n = (int)A.n, as_run = prm->as_run ? 1 : 0, min_nb = prm->min_neighbors;
    const double r = prm->radius;
    const PoseD cand = assess_candidate(prm, R_LI, T_LI);
    AsGrid L{};
    int cur = 0;
    long long records = n;
    if (leaf == 0.0) {
        *n_out = records;
        if (rec8 && cap < records) return fail(c, LIINIT_ERR_CAPACITY, "cap_records is smaller than the number of records");
        if (!rec8 && !out) return LIINIT_OK;
    } else {
        // the leaf grid first: a leaf too small for the cloud is refused before the moments run
        rc = assess_place(c, as_run, cand, leaf, true, L);
        if (rc) return rc;
        if (!rec8 && !out) {
            rc = assess_leaf_table(c, L, cur, records);
            if (rc) return rc;
            *n_out = records;
            return LIINIT_OK;
        }
    }
    // place and cell-sort once (the placement is the one above: same points, poses and extrinsics)
    AsGrid G;
    rc = assess_place(c, as_run, cand, assess_edge(r), false, G);
    if (rc) return rc;
    rc = assess_sort(c, G, cur);
    if (rc) return rc;
    k_as_gather<<<nblk(n, 256), 256, 0, c->stream>>>(A.world, A.key, A.v[cur], n, A.sorted, A.skey);
    c->launches++;
    CU(cudaGetLastError());
    // per-point n, h, v by stored index, in the sort buffers the gather has freed: A.v[0] (n ints), A.key and the A.k pair (one
    // allocation) as n doubles each. A.qn / A.qh / A.qv keep the last evaluation's values.
    int* pn = reinterpret_cast<int*>(A.v[0]);
    double* ph = reinterpret_cast<double*>(A.key);
    double* pv = reinterpret_cast<double*>(A.k[0]);
    const int nb = nblk(n, LI_FR_TILE);
    for (int a = 0; a < n; a += LI_AS_CLOUD_BATCH) {
        const int b = n - a > LI_AS_CLOUD_BATCH ? a + LI_AS_CLOUD_BATCH : n;   // the queries of this batch: stored points [a, b)
        k_as_mark<<<nb, LI_FR_TILE, 0, c->stream>>>(A.skey, A.sorted, n, 1, a, b, A.tc, A.tq);
        k_rs_scan<<<1, 1024, 0, c->stream>>>(nb + 1, A.tc);
        k_rs_scan<<<1, 1024, 0, c->stream>>>(nb + 1, A.tq);
        k_as_index<<<nb, LI_FR_TILE, 0, c->stream>>>(A.skey, A.sorted, n, 1, a, b, A.tc, A.tq, A.cell_start, A.cell_key, A.cell_q0, A.qlist);
        k_as_task_count<<<nb, LI_FR_TILE, 0, c->stream>>>(A.cell_q0, A.tc + nb, A.tt);
        k_rs_scan<<<1, 1024, 0, c->stream>>>(nb + 1, A.tt);
        k_as_task_emit<<<nb, LI_FR_TILE, 0, c->stream>>>(A.cell_q0, A.tc + nb, A.tt, A.tasks);
        c->launches += 7;
        CU(cudaGetLastError());
        CU(cudaMemsetAsync(A.ticket, 0, sizeof(unsigned), c->stream));
        k_as_moments<<<c->num_sms * 8, LI_AS_BLOCK, 0, c->stream>>>(A.sorted, A.cell_start, A.cell_key, A.tc + nb, A.qlist, A.tasks, A.tt + nb,
                                                                    A.ticket, G, r * r, 1, min_nb, pn, ph, pv);
        c->launches++;
        CU(cudaGetLastError());
    }
    k_as_reduce<<<1, 1024, 0, c->stream>>>(pn, ph, pv, n, min_nb, A.tot);
    c->launches++;
    CU(cudaGetLastError());
    AsTotals T;
    CU(cudaMemcpyAsync(&T, A.tot, sizeof(T), cudaMemcpyDeviceToHost, c->stream));
    if (leaf > 0.0) {
        // the record values of every point into A.sorted (free now), then the leaf sort (it reuses A.key, A.k, A.v)
        k_ac_point_pack<<<nblk(n, 256), 256, 0, c->stream>>>(ph, pv, pn, n, A.sorted);
        c->launches++;
        CU(cudaGetLastError());
        rc = assess_leaf_table(c, L, cur, records);
        if (rc) return rc;
        *n_out = records;
        if (rec8 && cap < records) return fail(c, LIINIT_ERR_CAPACITY, "cap_records is smaller than the number of records");
    } else {
        CU(cudaStreamSynchronize(c->stream));
    }
    if (out) {
        out->points = A.n;
        out->queries = A.n;
        out->stride = 1;
        out->scans = A.scans;
        out->valid = T.valid;
        out->sparse = T.sparse;
        out->degenerate = T.degenerate;
        out->mme = T.valid ? T.sum_h / (double)T.valid : NAN;
        out->mpv = T.valid ? T.sum_v / (double)T.valid : NAN;
    }
    if (!rec8) return LIINIT_OK;
    // the records reach the host in chunks through the strided staging buffer (free once a cloud is repacked)
    const long long chunk = (long long)(c->stage_raw_floats / 8);
    float4* stage = reinterpret_cast<float4*>(c->d_stage_raw);
    for (long long a = 0; a < records; a += chunk) {
        const int m = (int)(records - a < chunk ? records - a : chunk);
        if (leaf > 0.0)
            k_ac_leaf_rec<<<nblk(m, 256), 256, 0, c->stream>>>(A.world, A.sorted, A.v[cur], A.cell_start, (int)a, m, stage);
        else
            k_ac_point_rec<<<nblk(m, 256), 256, 0, c->stream>>>(A.world, ph, pv, pn, (int)a, m, stage);
        c->launches++;
        CU(cudaGetLastError());
        CU(cudaMemcpyAsync(rec8 + 8 * (size_t)a, stage, (size_t)m * 8 * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    }
    CU(cudaStreamSynchronize(c->stream));
    return LIINIT_OK;
}

}  // namespace

extern "C" {

}  // extern "C"

namespace {

// liinit_assess_reserve, and with max_pose_rows > 0 liinit_assess_reserve_timed
int assess_reserve(Ctx* c, long long max_points, int max_scans, long long max_pose_rows) {
    if (has_comm(c)) return fail(c, LIINIT_ERR_INVALID, "the map assessment does not take a communicator (liinit_comm_init)");
    if (max_points < 1 || max_points > LIINIT_ASSESS_MAX_POINTS) return fail(c, LIINIT_ERR_INVALID, "max_points must be in [1, LIINIT_ASSESS_MAX_POINTS]");
    if (max_scans < 1 || max_scans > LIINIT_ASSESS_MAX_SCANS) return fail(c, LIINIT_ERR_INVALID, "max_scans must be in [1, LIINIT_ASSESS_MAX_SCANS]");
    CU(cudaSetDevice(c->device));
    CU(cudaStreamSynchronize(c->stream));
    assess_free(c);
    Ctx::Assess& A = c->A;
    const size_t N = (size_t)max_points, Q = (size_t)(max_points < LIINIT_ASSESS_MAX_QUERIES ? max_points : LIINIT_ASSESS_MAX_QUERIES);
    const size_t NB = N / LI_FR_TILE + 2;
    bool ok = cudaMalloc(&A.pts, N * sizeof(float4)) == cudaSuccess && cudaMalloc(&A.poses, (size_t)max_scans * sizeof(PoseD)) == cudaSuccess &&
              cudaMalloc(&A.world, N * sizeof(float4)) == cudaSuccess && cudaMalloc(&A.sorted, N * sizeof(float4)) == cudaSuccess &&
              cudaMalloc(&A.key, N * 8) == cudaSuccess && cudaMalloc(&A.skey, N * 8) == cudaSuccess && cudaMalloc(&A.k[0], N * 8) == cudaSuccess &&
              cudaMalloc(&A.v[0], N * 4) == cudaSuccess && cudaMalloc(&A.v[1], N * 4) == cudaSuccess &&
              cudaMalloc(&A.hist, (N / RS_TILE + 2) * 256 * 4) == cudaSuccess && cudaMalloc(&A.tc, NB * 4) == cudaSuccess &&
              cudaMalloc(&A.tq, NB * 4) == cudaSuccess && cudaMalloc(&A.tt, NB * 4) == cudaSuccess && cudaMalloc(&A.cell_start, (N + 1) * 4) == cudaSuccess &&
              cudaMalloc(&A.cell_key, N * 8) == cudaSuccess && cudaMalloc(&A.cell_q0, (N + 1) * 4) == cudaSuccess && cudaMalloc(&A.qlist, Q * 4) == cudaSuccess &&
              cudaMalloc(&A.tasks, Q * sizeof(int4)) == cudaSuccess && cudaMalloc(&A.qn, Q * 4) == cudaSuccess && cudaMalloc(&A.qh, Q * 8) == cudaSuccess &&
              cudaMalloc(&A.qv, Q * 8) == cudaSuccess && cudaMalloc(&A.box, 8 * 4) == cudaSuccess && cudaMalloc(&A.tot, sizeof(AsTotals)) == cudaSuccess &&
              cudaMalloc(&A.ticket, sizeof(unsigned)) == cudaSuccess;
    if (ok && max_pose_rows > 0)
        ok = cudaMalloc(&A.raw, N * sizeof(float4)) == cudaSuccess && cudaMalloc(&A.at, (size_t)max_scans * sizeof(AtScan)) == cudaSuccess &&
             cudaMalloc(&A.at_end, (size_t)max_scans * sizeof(PoseD)) == cudaSuccess &&
             cudaMalloc(&A.pool, (size_t)max_pose_rows * LI_POSE6D_DOUBLES * sizeof(double)) == cudaSuccess;
    if (ok) A.k[1] = A.k[0] + N;   // one allocation: a cloud keeps n doubles in it (assess_cloud)
    if (!ok) {
        cudaGetLastError();
        assess_free(c);
        return fail(c, LIINIT_ERR_CUDA, "cudaMalloc of the assessment store (" + std::to_string(max_points) + " points) failed");
    }
    A.cap = max_points;
    A.max_scans = max_scans;
    A.timed = max_pose_rows > 0;
    A.pool_cap = max_pose_rows;
    return LIINIT_OK;
}

// the store of liinit_assess_append (k_as_store) for a staged cloud that fits; a timed store also records the scan's timing (timing
// NULL: an untimed scan)
int assess_store(Ctx* c, const double* rot_end, const double* pos_end, const double* R_LI, const double* T_LI, const AtScan* timing = nullptr) {
    Ctx::Assess& A = c->A;
    PoseD P;
    fill_pose(P, rot_end, pos_end, R_LI, T_LI);
    if (A.timed) {
        const AtScan untimed{};   // npose = 0
        CU(cudaMemcpyAsync(A.at + A.scans, timing ? timing : &untimed, sizeof(AtScan), cudaMemcpyHostToDevice, c->stream));
        if (timing) A.timed_scans++; else A.untimed_scans++;
    }
    k_as_store<<<nblk(c->raw_n, 256), 256, 0, c->stream>>>(c->d_stage_pts, c->raw_n, A.scans, P, A.pts + A.n, A.poses);
    c->launches++;
    CU(cudaGetLastError());
    A.n += c->raw_n;
    A.scans++;
    A.hold_seq = -1;
    return LIINIT_OK;
}

}  // namespace

extern "C" {

int liinit_assess_reserve(liinit_ctx* h, long long max_points, int max_scans) {
    if (!h) return LIINIT_ERR_INVALID;
    return assess_reserve(&h->c, max_points, max_scans, 0);
}

int liinit_assess_reserve_timed(liinit_ctx* h, long long max_points, int max_scans, long long max_pose_rows) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    if (max_pose_rows < 2 || max_pose_rows > LIINIT_ASSESS_MAX_POSE_ROWS)
        return fail(c, LIINIT_ERR_INVALID, "max_pose_rows must be in [2, LIINIT_ASSESS_MAX_POSE_ROWS]");
    return assess_reserve(c, max_points, max_scans, max_pose_rows);
}

int liinit_assess_append(liinit_ctx* h, const double rot_end[9], const double pos_end[3], const double R_LI[9], const double T_LI[3],
                         int* appended) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    if (!rot_end || !pos_end || !R_LI || !T_LI || !appended) return fail(c, LIINIT_ERR_INVALID, "null argument");
    int r = assess_check(c);
    if (r) return r;
    if (c->raw_n <= 0) return fail(c, LIINIT_ERR_INVALID, "no raw cloud staged (liinit_raw_upload / liinit_frame_stage)");
    CU(cudaSetDevice(c->device));
    Ctx::Assess& A = c->A;
    if (A.n + c->raw_n > A.cap || A.scans >= A.max_scans) {
        A.skipped++;
        *appended = 0;
        return LIINIT_OK;
    }
    r = assess_store(c, rot_end, pos_end, R_LI, T_LI);
    if (r) return r;
    *appended = 1;
    return LIINIT_OK;
}

int liinit_assess_hold(liinit_ctx* h) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    int r = assess_check(c);
    if (r) return r;
    Ctx::Assess& A = c->A;
    if (!A.timed) return fail(c, LIINIT_ERR_INVALID, "the assessment store is not timed (liinit_assess_reserve_timed)");
    if (c->raw_n <= 0) return fail(c, LIINIT_ERR_INVALID, "no raw cloud staged (liinit_raw_upload / liinit_frame_stage)");
    CU(cudaSetDevice(c->device));
    // a cloud the store has no room for is not copied: its append is skipped
    if (A.n + c->raw_n <= A.cap)
        CU(cudaMemcpyAsync(A.raw + A.n, c->d_stage_pts, (size_t)c->raw_n * sizeof(float4), cudaMemcpyDeviceToDevice, c->stream));
    A.hold_seq = c->stage_seq;
    A.hold_n = c->raw_n;
    A.hold_at = A.n;
    return LIINIT_OK;
}

int liinit_assess_append_timed(liinit_ctx* h, const double rot_end[9], const double pos_end[3], const double R_LI[9], const double T_LI[3],
                               const liinit_assess_timing* t, int* appended) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    if (!rot_end || !pos_end || !R_LI || !T_LI || !t || !appended) return fail(c, LIINIT_ERR_INVALID, "null argument");
    int r = assess_check(c);
    if (r) return r;
    Ctx::Assess& A = c->A;
    if (!A.timed) return fail(c, LIINIT_ERR_INVALID, "the assessment store is not timed (liinit_assess_reserve_timed)");
    if (c->raw_n <= 0) return fail(c, LIINIT_ERR_INVALID, "no raw cloud staged (liinit_raw_upload / liinit_frame_stage)");
    if (A.hold_seq != c->stage_seq || A.hold_at != A.n)
        return fail(c, LIINIT_ERR_INVALID, "no hold of the staged cloud (liinit_assess_hold after staging it, before the undistortion)");
    if (A.hold_n != c->raw_n) return fail(c, LIINIT_ERR_INVALID, "the held cloud and the staged cloud differ in size");
    if (t->npose < 2 || t->npose > LIINIT_MAX_IMU_POSES) return fail(c, LIINIT_ERR_INVALID, "npose must be in [2, LIINIT_MAX_IMU_POSES]");
    if (!t->poses) return fail(c, LIINIT_ERR_INVALID, "null pose table");
    CU(cudaSetDevice(c->device));
    if (A.n + c->raw_n > A.cap || A.scans >= A.max_scans) {
        A.skipped++;
        A.hold_seq = -1;
        *appended = 0;
        return LIINIT_OK;
    }
    if (A.pool_rows + t->npose > A.pool_cap) {   // no room for the table: stored as an untimed scan
        r = assess_store(c, rot_end, pos_end, R_LI, T_LI);
        if (r) return r;
        *appended = 1;
        return LIINIT_OK;
    }
    AtScan s{};
    fill_pose(s.prior, t->rot, t->pos, t->R_LI, t->T_LI);
    memcpy(s.vel, t->vel, 24);
    s.row0 = A.pool_rows;
    s.npose = t->npose;
    CU(cudaMemcpyAsync(A.pool + (size_t)A.pool_rows * LI_POSE6D_DOUBLES, t->poses, (size_t)t->npose * LI_POSE6D_DOUBLES * sizeof(double),
                       cudaMemcpyHostToDevice, c->stream));
    A.pool_rows += t->npose;
    r = assess_store(c, rot_end, pos_end, R_LI, T_LI, &s);
    if (r) return r;
    *appended = 1;
    return LIINIT_OK;
}

int liinit_assess_timing_info(liinit_ctx* h, int* timed_scans, int* untimed_scans, long long* pose_rows) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    int r = assess_check(c);
    if (r) return r;
    if (!c->A.timed) return fail(c, LIINIT_ERR_INVALID, "the assessment store is not timed (liinit_assess_reserve_timed)");
    if (timed_scans) *timed_scans = c->A.timed_scans;
    if (untimed_scans) *untimed_scans = c->A.untimed_scans;
    if (pose_rows) *pose_rows = c->A.pool_rows;
    return LIINIT_OK;
}

int liinit_assess_info(liinit_ctx* h, long long* points, int* scans, int* skipped) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    int r = assess_check(c);
    if (r) return r;
    if (points) *points = c->A.n;
    if (scans) *scans = c->A.scans;
    if (skipped) *skipped = c->A.skipped;
    return LIINIT_OK;
}

int liinit_assess_evaluate(liinit_ctx* h, const liinit_assess_params* p, const double R_LI[9], const double T_LI[3], liinit_assess_result* out) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    if (!p || !out) return fail(c, LIINIT_ERR_INVALID, "null argument");
    int r = assess_check(c);
    if (r) return r;
    CU(cudaSetDevice(c->device));
    return assess_evaluate(c, p, R_LI, T_LI, out);
}

int liinit_assess_evaluate_timed(liinit_ctx* h, const liinit_assess_params* p, const double R_LI[9], const double T_LI[3], double lag_shift,
                                 liinit_assess_result* out) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    if (!p || !out) return fail(c, LIINIT_ERR_INVALID, "null argument");
    int r = assess_check(c);
    if (r) return r;
    if (!c->A.timed) return fail(c, LIINIT_ERR_INVALID, "the assessment store is not timed (liinit_assess_reserve_timed)");
    if (!std::isfinite(lag_shift)) return fail(c, LIINIT_ERR_INVALID, "lag_shift must be finite");
    CU(cudaSetDevice(c->device));
    return assess_evaluate(c, p, R_LI, T_LI, out, &lag_shift);
}

int liinit_assess_cloud(liinit_ctx* h, const liinit_assess_params* p, const double R_LI[9], const double T_LI[3], double leaf, float* rec8,
                        long long cap_records, long long* n, liinit_assess_result* totals) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    if (!p || !n) return fail(c, LIINIT_ERR_INVALID, "null argument");
    int r = assess_check(c);
    if (r) return r;
    CU(cudaSetDevice(c->device));
    return assess_cloud(c, p, R_LI, T_LI, leaf, rec8, cap_records, n, totals);
}

int liinit_assess_download(liinit_ctx* h, double* h_out, double* v_out, int* n_out, long long cap, long long* n) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    if (!n) return fail(c, LIINIT_ERR_INVALID, "null argument");
    int r = assess_check(c);
    if (r) return r;
    const long long q = c->A.last_q;
    if (q < 0) return fail(c, LIINIT_ERR_INVALID, "no evaluation since the store was reserved (liinit_assess_evaluate)");
    *n = q;
    if ((h_out || v_out || n_out) && cap < q) return fail(c, LIINIT_ERR_CAPACITY, "cap is smaller than the number of queries");
    CU(cudaSetDevice(c->device));
    if (h_out) CU(cudaMemcpyAsync(h_out, c->A.qh, (size_t)q * 8, cudaMemcpyDeviceToHost, c->stream));
    if (v_out) CU(cudaMemcpyAsync(v_out, c->A.qv, (size_t)q * 8, cudaMemcpyDeviceToHost, c->stream));
    if (n_out) CU(cudaMemcpyAsync(n_out, c->A.qn, (size_t)q * 4, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return LIINIT_OK;
}

int liinit_assess_download_placed(liinit_ctx* h, float* xyz, long long cap, long long* n) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    if (!n) return fail(c, LIINIT_ERR_INVALID, "null argument");
    int r = assess_check(c);
    if (r) return r;
    if (c->A.last_q < 0) return fail(c, LIINIT_ERR_INVALID, "no evaluation since the store was reserved (liinit_assess_evaluate)");
    const long long m = c->A.last_n;
    *n = m;
    if (!xyz) return LIINIT_OK;
    if (cap < m) return fail(c, LIINIT_ERR_CAPACITY, "cap is smaller than the number of stored points");
    CU(cudaSetDevice(c->device));
    return download_xyz(c, c->A.world, (size_t)m, xyz);
}

}  // extern "C"

namespace {

// cudaMalloc that first frees what p held (a snapshot buffer that has to grow)
template <class T>
cudaError_t regrow(T*& p, size_t count) {
    cudaFree(p);
    p = nullptr;
    return cudaMalloc(&p, count * sizeof(T));
}

// the replay store a context reads: its lead's while it shares one (liinit_replay_share), else its own
const Ctx::Replay& replay_store(const Ctx* c) { return c->share_lead ? c->share_lead->R : c->R; }

// the calls that change a replay store or a map snapshot are refused on a worker and on a lead with workers
int refuse_shared(Ctx* c, const char* what) {
    if (c->share_lead) return fail(c, LIINIT_ERR_INVALID, std::string(what) + " on a context that shares a lead's replay store (liinit_replay_unshare it first)");
    if (c->share_workers.load() > 0)
        return fail(c, LIINIT_ERR_INVALID, std::string(what) + " on a context whose replay store and map snapshot workers share (liinit_replay_unshare them first)");
    return LIINIT_OK;
}

int map_snapshot(Ctx* c, long long* bytes) {
    int r = fetch_counters(c);   // (synchronises: the host mirrors and the counts that size the copies are current)
    if (r) return r;
    Ctx::Snap& S = c->snap;
    const size_t slots = c->hash_slots;
    const unsigned long long top = *c->h_pool_top;
    const int bricks = c->h_counters[CNT_BRICKS];
    bool ok = true;
    if (!S.ent) {
        ok = cudaMalloc(&S.ent, slots * sizeof(uint4)) == cudaSuccess && cudaMalloc(&S.aux, slots * sizeof(uint4)) == cudaSuccess &&
             cudaMalloc(&S.brick_slots, slots * sizeof(int)) == cudaSuccess &&
             cudaMalloc(&S.counters, CNT_COUNT * sizeof(int) + sizeof(unsigned long long)) == cudaSuccess;
        if (ok && c->cells)
            ok = cudaMalloc(&S.cocc, slots * 8) == cudaSuccess && cudaMalloc(&S.cdir, slots * 64 * sizeof(unsigned short)) == cudaSuccess &&
                 cudaMalloc(&S.sb_keys, slots * 8) == cudaSuccess && cudaMalloc(&S.sb_occ, slots * 8) == cudaSuccess;
    }
    if (ok && top > S.pool_alloc) {
        ok = regrow(S.pool, (size_t)top) == cudaSuccess;
        S.pool_alloc = ok ? top : 0;
    }
    if (ok && c->raw_n > S.stage_alloc) {
        ok = regrow(S.stage_pts, (size_t)c->raw_n) == cudaSuccess && regrow(S.stage_attr, (size_t)c->raw_n) == cudaSuccess;
        S.stage_alloc = ok ? c->raw_n : 0;
    }
    if (!ok) {
        cudaGetLastError();
        snap_free(c);
        return fail(c, LIINIT_ERR_CUDA, "cudaMalloc of the map snapshot failed");
    }
    long long b = 0;
    auto d2d = [&](void* dst, const void* src, size_t n) {
        b += (long long)n;
        return n ? cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToDevice, c->stream) : cudaSuccess;
    };
    CU(d2d(S.ent, c->M.ent, slots * sizeof(uint4)));
    CU(d2d(S.aux, c->M.aux, slots * sizeof(uint4)));
    CU(d2d(S.brick_slots, c->M.brick_slots, (size_t)bricks * sizeof(int)));
    CU(d2d(S.counters, c->d_counters, CNT_COUNT * sizeof(int)));
    CU(d2d(S.counters + CNT_COUNT, c->M.pool_top, sizeof(unsigned long long)));
    CU(d2d(S.pool, c->M.pool, (size_t)top * sizeof(float4)));
    if (c->cells) {
        CU(d2d(S.cocc, c->M.cocc, slots * 8));
        CU(d2d(S.cdir, c->M.cdir, slots * 64 * sizeof(unsigned short)));
        CU(d2d(S.sb_keys, c->M.sb_keys, slots * 8));
        CU(d2d(S.sb_occ, c->M.sb_occ, slots * 8));
    }
    CU(d2d(S.stage_pts, c->d_stage_pts, (size_t)c->raw_n * sizeof(float4)));
    if (c->stage_attr) CU(d2d(S.stage_attr, c->d_stage_attr, (size_t)c->raw_n * sizeof(float4)));
    memcpy(S.h_counters, c->h_counters, sizeof(S.h_counters));
    S.pool_top = top;
    S.raw_n = c->raw_n;
    S.stage_attr_on = c->stage_attr;
    S.have = true;
    if (bytes) *bytes = b;
    return LIINIT_OK;
}

int map_restore(Ctx* c) {
    const Ctx::Snap& S = c->share_lead ? c->share_lead->snap : c->snap;
    if (!S.have) return fail(c, LIINIT_ERR_INVALID, "no map snapshot (liinit_map_snapshot)");
    const size_t slots = c->hash_slots;
    auto d2d = [&](void* dst, const void* src, size_t n) {
        return n ? cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToDevice, c->stream) : cudaSuccess;
    };
    CU(d2d(c->M.ent, S.ent, slots * sizeof(uint4)));
    CU(d2d(c->M.aux, S.aux, slots * sizeof(uint4)));
    CU(d2d(c->M.brick_slots, S.brick_slots, (size_t)S.h_counters[CNT_BRICKS] * sizeof(int)));
    CU(d2d(c->d_counters, S.counters, CNT_COUNT * sizeof(int)));
    CU(d2d(c->M.pool_top, S.counters + CNT_COUNT, sizeof(unsigned long long)));
    CU(d2d(c->M.pool, S.pool, (size_t)S.pool_top * sizeof(float4)));
    if (c->cells) {
        CU(d2d(c->M.cocc, S.cocc, slots * 8));
        CU(d2d(c->M.cdir, S.cdir, slots * 64 * sizeof(unsigned short)));
        CU(d2d(c->M.sb_keys, S.sb_keys, slots * 8));
        CU(d2d(c->M.sb_occ, S.sb_occ, slots * 8));
    }
    CU(d2d(c->d_stage_pts, S.stage_pts, (size_t)S.raw_n * sizeof(float4)));
    if (S.stage_attr_on) CU(d2d(c->d_stage_attr, S.stage_attr, (size_t)S.raw_n * sizeof(float4)));
    memcpy(c->h_counters, S.h_counters, sizeof(S.h_counters));
    *c->h_pool_top = S.pool_top;
    c->map_epoch++;   // the restore can remove map points
    c->raw_n = S.raw_n;
    c->stage_attr = S.stage_attr_on;
    c->stage_seq++;
    return LIINIT_OK;
}

}  // namespace

extern "C" {

int liinit_assess_clear(liinit_ctx* h) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    int r = assess_check(c);
    if (r) return r;
    Ctx::Assess& A = c->A;
    A.n = 0;
    A.scans = A.skipped = 0;
    A.last_q = -1;
    A.last_n = 0;
    A.timed_scans = A.untimed_scans = 0;
    A.pool_rows = 0;
    A.hold_seq = -1;
    return LIINIT_OK;
}

int liinit_map_snapshot(liinit_ctx* h, long long* bytes) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    if (has_comm(c)) return fail(c, LIINIT_ERR_INVALID, "the map snapshot does not take a communicator (liinit_comm_init)");
    int r = refuse_shared(c, "liinit_map_snapshot");
    if (r) return r;
    CU(cudaSetDevice(c->device));
    return map_snapshot(c, bytes);
}

int liinit_map_restore(liinit_ctx* h) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    CU(cudaSetDevice(c->device));
    return map_restore(c);
}

int liinit_replay_reserve(liinit_ctx* h, long long max_points, int max_frames) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    if (max_points < 1 || max_points > LIINIT_ASSESS_MAX_POINTS) return fail(c, LIINIT_ERR_INVALID, "max_points must be in [1, LIINIT_ASSESS_MAX_POINTS]");
    if (max_frames < 1 || max_frames > LIINIT_ASSESS_MAX_SCANS) return fail(c, LIINIT_ERR_INVALID, "max_frames must be in [1, LIINIT_ASSESS_MAX_SCANS]");
    int r = refuse_shared(c, "liinit_replay_reserve");
    if (r) return r;
    CU(cudaSetDevice(c->device));
    CU(cudaStreamSynchronize(c->stream));
    replay_free(c);
    Ctx::Replay& R = c->R;
    if (cudaMalloc(&R.pts, (size_t)max_points * sizeof(float4)) != cudaSuccess || cudaMalloc(&R.inten, (size_t)max_points * sizeof(float)) != cudaSuccess) {
        cudaGetLastError();
        replay_free(c);
        return fail(c, LIINIT_ERR_CUDA, "cudaMalloc of the replay store (" + std::to_string(max_points) + " points) failed");
    }
    R.cap = max_points;
    R.max_frames = max_frames;
    R.fr.reserve((size_t)(max_frames < 65536 ? max_frames : 65536));
    return LIINIT_OK;
}

int liinit_replay_append(liinit_ctx* h, long long handle, double t_beg, float end_ms, int* appended) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    if (!appended) return fail(c, LIINIT_ERR_INVALID, "null argument");
    int r = refuse_shared(c, "liinit_replay_append");
    if (r) return r;
    Ctx::Replay& R = c->R;
    if (R.cap <= 0) return fail(c, LIINIT_ERR_INVALID, "no replay store (liinit_replay_reserve)");
    int slot = 0;
    const FrameSub* s = frame_lookup(c, handle, &slot);
    if (!s) return fail(c, LIINIT_ERR_INVALID, "unknown sub-frame handle (its message slot has been reused)");
    CU(cudaSetDevice(c->device));
    if (R.n + s->n > R.cap || (int)R.fr.size() >= R.max_frames) {
        R.skipped++;
        *appended = 0;
        return LIINIT_OK;
    }
    const size_t o = (size_t)slot * c->stage_pts_cap + (s->lo - 1);
    CU(cudaMemcpyAsync(R.pts + R.n, c->d_fr_slot_pts + o, (size_t)s->n * sizeof(float4), cudaMemcpyDeviceToDevice, c->stream));
    CU(cudaMemcpyAsync(R.inten + R.n, c->d_fr_slot_inten + o, (size_t)s->n * sizeof(float), cudaMemcpyDeviceToDevice, c->stream));
    R.fr.push_back(Ctx::ReplayFrame{t_beg, end_ms, s->n, R.n});
    R.n += s->n;
    *appended = 1;
    return LIINIT_OK;
}

int liinit_replay_info(liinit_ctx* h, int* frames, int* skipped, long long* points) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    const Ctx::Replay& R = replay_store(c);
    if (R.cap <= 0) return fail(c, LIINIT_ERR_INVALID, "no replay store (liinit_replay_reserve)");
    if (frames) *frames = (int)R.fr.size();
    if (skipped) *skipped = R.skipped;
    if (points) *points = R.n;
    return LIINIT_OK;
}

int liinit_replay_frame(liinit_ctx* h, int j, double* t_beg, float* end_ms, int* n) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    const Ctx::Replay& R = replay_store(c);
    if (j < 0 || j >= (int)R.fr.size()) return fail(c, LIINIT_ERR_INVALID, "no such stored sub-frame");
    const Ctx::ReplayFrame& f = R.fr[j];
    if (t_beg) *t_beg = f.t_beg;
    if (end_ms) *end_ms = f.end_ms;
    if (n) *n = f.n;
    return LIINIT_OK;
}

int liinit_replay_stage(liinit_ctx* h, int j) {
    if (!h) return LIINIT_ERR_INVALID;
    Ctx* c = &h->c;
    const Ctx::Replay& R = replay_store(c);
    if (j < 0 || j >= (int)R.fr.size()) return fail(c, LIINIT_ERR_INVALID, "no such stored sub-frame");
    CU(cudaSetDevice(c->device));
    const Ctx::ReplayFrame& f = R.fr[j];
    // liinit_frame_stage's copy and attribute kernel, from the store instead of the message slot
    CU(cudaMemcpyAsync(c->d_stage_pts, R.pts + f.lo, (size_t)f.n * sizeof(float4), cudaMemcpyDeviceToDevice, c->stream));
    k_attr_from_inten<<<nblk(f.n, 256), 256, 0, c->stream>>>(R.inten + f.lo, f.n, c->d_stage_attr);
    c->launches++;
    CU(cudaGetLastError());
    c->stage_attr = true;
    c->raw_n = f.n;
    c->stage_seq++;
    return LIINIT_OK;
}

int liinit_replay_share(liinit_ctx* worker, liinit_ctx* lead) {
    if (!worker) return LIINIT_ERR_INVALID;
    Ctx* c = &worker->c;
    if (!lead) return fail(c, LIINIT_ERR_INVALID, "null lead");
    Ctx* L = &lead->c;
    if (worker == lead) return fail(c, LIINIT_ERR_INVALID, "a context cannot share its own replay store");
    if (c->device != L->device) return fail(c, LIINIT_ERR_INVALID, "the worker and the lead are on different devices");
    if (c->hash_slots != L->hash_slots || c->M.bshift != L->M.bshift || c->cells != L->cells || c->M.pool_cap != L->M.pool_cap ||
        c->stage_pts_cap != L->stage_pts_cap || c->cfg.max_map_points != L->cfg.max_map_points || c->cfg.max_scan_points != L->cfg.max_scan_points ||
        c->M.ds != L->M.ds)
        return fail(c, LIINIT_ERR_INVALID, "the worker's configuration differs from the lead's (hash slots, brick cells, cell directory, "
                                           "capacities or filter_size_map)");
    if (has_comm(c) || has_comm(L)) return fail(c, LIINIT_ERR_INVALID, "replay sharing does not take a communicator (liinit_comm_init)");
    if (c->share_lead) return fail(c, LIINIT_ERR_INVALID, "the worker already shares a lead's replay store");
    if (c->share_workers.load() > 0) return fail(c, LIINIT_ERR_INVALID, "the worker is itself the lead of other workers");
    if (L->share_lead) return fail(c, LIINIT_ERR_INVALID, "the lead shares another context's replay store");
    if (!L->snap.have) return fail(c, LIINIT_ERR_INVALID, "the lead has no map snapshot (liinit_map_snapshot)");
    if (L->R.cap <= 0) return fail(c, LIINIT_ERR_INVALID, "the lead has no replay store (liinit_replay_reserve)");
    CU(cudaSetDevice(L->device));
    CU(cudaStreamSynchronize(L->stream));   // the store and the snapshot are complete before any worker's stream reads them
    c->share_lead = L;
    L->share_workers++;
    return LIINIT_OK;
}

int liinit_replay_unshare(liinit_ctx* worker) {
    if (!worker) return LIINIT_ERR_INVALID;
    Ctx* c = &worker->c;
    if (!c->share_lead) return fail(c, LIINIT_ERR_INVALID, "the context does not share a lead's replay store");
    CU(cudaSetDevice(c->device));
    CU(cudaStreamSynchronize(c->stream));   // its reads of the lead's store and snapshot are done
    c->share_lead->share_workers--;
    c->share_lead = nullptr;
    return LIINIT_OK;
}

}  // extern "C"
