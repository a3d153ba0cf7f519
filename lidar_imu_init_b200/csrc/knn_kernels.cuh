// knn_kernels.cuh -- exact bounded 5-NN on the brick hash (replaces KD_TREE::Nearest_Search,
// ikd_Tree.cpp:349-379, Search :825-968).
//
// G lanes (G = 2, 4, 8, 16 or 32; chosen per pass from the frame size, group_for() in liinit_gpu.cu) cooperate on one query, so a warp works on Q = 32/G queries AT ONCE and IN LOCKSTEP:
// every loop is warp-uniform (its trip count is the maximum over the warp's groups, idle groups are predicated
// off) and every shuffle / ballot uses the full mask. Sub-mask *_sync intrinsics make the hardware run the groups
// one after the other (measured in round 1: 11 of 32 lanes active); lockstep keeps all 32 lanes issuing together.
//
//   Shell iteration on the brick-box distance (see knn5_lockstep): the first shell is a guessed radius rho around the
//   query, then one closing shell [rho^2, g5) once 5 neighbours are known (or growing shells while fewer are known).
//   The search is exact: it stops only when no unscanned brick can hold a point closer than the current 5th.
//   Inside a shell every brick is probed first (two hash probes in flight per lane, found bricks listed per group in shared memory),
//   then the listed slabs are scanned slot-aligned: the s-th brick of every group at the same time.
//
// A brick's slab is read by G consecutive lanes -> contiguous 16*G-byte segments; every lane keeps a private sorted
// top-5 of the candidates IT saw; the group's top-5 is merged at phase boundaries.
// Semantics matched (DESIGN.md section 3): candidates with d2 <= 5 only (ikd_Tree.cpp:842, sic), fp32
// (dx*dx+dy*dy)+dz*dz without FMA, ascending output; exact-tie handling is traversal dependent in the
// reference and therefore excluded from the parity claim.
#pragma once
#include "common.cuh"

#ifndef LI_KNN_U
#define LI_KNN_U 2           // slab loads issued back to back per lane before the distances are evaluated (H100 sweep, DESIGN section 3)
#endif
#ifndef LI_KNN_THREADS
#define LI_KNN_THREADS 128
#endif
#ifndef LI_KNN_MIN_BLOCKS
#define LI_KNN_MIN_BLOCKS 8   // resident blocks per SM the search kernel is compiled for (register budget)
#endif

template <int G>
struct Grp {
    static constexpr int Q = 32 / G;
    static constexpr unsigned GM = (G == 32) ? 0xffffffffu : ((1u << G) - 1u);
};

// ---- full-mask group primitives (all 32 lanes must call) -------------------------------------------------
template <int G>
__device__ __forceinline__ unsigned grp_ballot(bool p, int gbase) {
    return (__ballot_sync(LI_FULL, p) >> gbase) & Grp<G>::GM;
}
template <int G, class T>
__device__ __forceinline__ T grp_shfl(T v, int src_rel, int gbase) {
    return __shfl_sync(LI_FULL, v, gbase + src_rel);
}
template <int G>
__device__ __forceinline__ unsigned grp_min(unsigned v) {
    if constexpr (G == 32) {
        return __reduce_min_sync(LI_FULL, v);
    } else {
#pragma unroll
        for (int o = G / 2; o >= 1; o >>= 1) v = min(v, __shfl_xor_sync(LI_FULL, v, o));
        return v;
    }
}

// sorted insert into a lane-private top-5 (precondition: d < ld[4]); stable w.r.t. equal distances
__device__ __forceinline__ void local_insert(float (&ld)[5], int (&li)[5], float d, int id) {
    ld[4] = d;
    li[4] = id;
#pragma unroll
    for (int i = 4; i > 0; --i) {
        bool sw = ld[i] < ld[i - 1];
        float a = ld[i - 1], b = ld[i];
        int ia = li[i - 1], ib = li[i];
        ld[i - 1] = sw ? b : a;
        ld[i] = sw ? a : b;
        li[i - 1] = sw ? ib : ia;
        li[i] = sw ? ia : ib;
    }
}

// Group-wide top-5 of the G private lists -> gd/gi (uniform in the group).
template <int G>
__device__ __forceinline__ void group_merge(const float (&ld)[5], const int (&li)[5], float (&gd)[5], int (&gi)[5], int gl, int gbase) {
    float cd[5];
    int ci[5];
#pragma unroll
    for (int i = 0; i < 5; i++) {
        cd[i] = ld[i];
        ci[i] = li[i];
    }
#pragma unroll
    for (int k = 0; k < 5; k++) {
        unsigned hb = __float_as_uint(cd[0]);
        unsigned mn = grp_min<G>(hb);
        unsigned who = grp_ballot<G>(hb == mn, gbase);
        int src = __ffs(who) - 1;
        gd[k] = __uint_as_float(mn);
        gi[k] = grp_shfl<G>(ci[0], src, gbase);
        if (gl == src) {
#pragma unroll
            for (int i = 0; i < 4; i++) {
                cd[i] = cd[i + 1];
                ci[i] = ci[i + 1];
            }
            cd[4] = INFINITY;
            ci[4] = -1;
        }
    }
}

// Lockstep scan of one slab per group (cnt = 0 for idle groups). U loads are issued back to back before any distance
// is evaluated and the NEXT batch is already in flight while the current one is processed (double buffering), so the
// L2 round trips overlap with the arithmetic. One compare per candidate: tau = min(thr, 5+, lane's 5th best).
//
// Shape of the loop (from the SASS of the first version: 64-bit address
// arithmetic per load, three padding moves per candidate and twelve register moves per iteration to rotate the
// buffers made up a third of the loop):
//   * one running pointer per lane, the 2U loads of a round use constant offsets from it;
//   * out-of-range slots are not padded: the load is predicated (the register keeps an old, finite point) and the
//     range test is folded into the candidate's single compare;
//   * the two buffers swap roles by unrolling the loop twice instead of being copied.
// (sm_90 has no packed fp32 pipe, so the candidate distance is the scalar li_dist2.)
// a float the compiler must treat as defined but that costs no instruction (contents: whatever the register held)
__device__ __forceinline__ float li_stale_float() {
#ifdef LI_SIMT_EMUL
    return 0.f;
#else
    float v;
    asm("" : "=f"(v));
    return v;
#endif
}
// One buffered candidate: its xyz only. A 128-bit load would tie up the never-read voxel-id word as a fourth register for as long
// as the candidate waits in the buffer; an 8-byte + a 4-byte load keep three (and measured faster on H100, DESIGN section 3).
struct LiXyz {
    float2 xy;
    float z;
};
__device__ __forceinline__ void li_load_xyz(const float4* __restrict__ p, LiXyz& c) {
    c.xy = __ldg(reinterpret_cast<const float2*>(p));
    c.z = __ldg(reinterpret_cast<const float*>(p) + 2);
}
template <int G, int U = LI_KNN_U>
__device__ __forceinline__ void group_scan_pipelined(const float4* __restrict__ pool, unsigned f, unsigned cnt, float qx, float qy, float qz,
                                                     float thr, float (&ld)[5], int (&li)[5], int gl) {
    const float cap5 = __uint_as_float(0x40a00001u);   // smallest float above 5: d <= 5 <=> d < cap5
    const float thr5 = fminf(thr, cap5);
    float tau = fminf(thr5, ld[4]);
    const float4* __restrict__ ptr = pool + f + gl;    // this lane's next candidate; the 2U loads of a round use constant offsets from it
    int rem = (int)cnt - gl;                            // candidates left for this lane's column, in units of slab slots
    LiXyz a[U], b[U];
#pragma unroll
    for (int u = 0; u < U; u++) {   // slots never loaded are never used: their compare is masked by the range test
        a[u].xy = make_float2(li_stale_float(), li_stale_float());
        a[u].z = li_stale_float();
        b[u].xy = make_float2(li_stale_float(), li_stale_float());
        b[u].z = li_stale_float();
    }
#pragma unroll
    for (int u = 0; u < U; u++)
        if (u * G < rem) li_load_xyz(ptr + u * G, a[u]);
    while (__any_sync(LI_FULL, rem > 0)) {
#pragma unroll
        for (int u = 0; u < U; u++)
            if ((U + u) * G < rem) li_load_xyz(ptr + (U + u) * G, b[u]);
#pragma unroll
        for (int u = 0; u < U; u++) {
            float d = li_dist2(qx, qy, qz, a[u].xy.x, a[u].xy.y, a[u].z);
            if (d < tau && u * G < rem) {
                local_insert(ld, li, d, (int)(ptr - pool) + u * G);   // (the pool offset: only formed for an insert)
                tau = fminf(thr5, ld[4]);
            }
        }
        if (!__any_sync(LI_FULL, rem > U * G)) break;
#pragma unroll
        for (int u = 0; u < U; u++)
            if ((2 * U + u) * G < rem) li_load_xyz(ptr + (2 * U + u) * G, a[u]);
#pragma unroll
        for (int u = 0; u < U; u++) {
            float d = li_dist2(qx, qy, qz, b[u].xy.x, b[u].xy.y, b[u].z);
            if (d < tau && (U + u) * G < rem) {
                local_insert(ld, li, d, (int)(ptr - pool) + (U + u) * G);
                tau = fminf(thr5, ld[4]);
            }
        }
        ptr += 2 * U * G;
        rem -= 2 * U * G;
    }
}

__device__ __forceinline__ int li_shl(int v, int s) { return (int)((unsigned)v << s); }   // v * 2^s for either sign

struct KnnGeom {
    int bs;             // log2(voxels per brick edge)
    float ds, margin;   // voxel edge; rounding slack added to every pruning box
};

// ---- a shell: PROBE ALL its bricks first, then scan what was found SLOT-ALIGNED -------------------------------------------------------
// Round 1 alternated {enumerate G bricks, probe them, scan what was found}: a 27-brick closing shell was seven dependent
// {hash probe -> slab loads} round trips, and in most of those rounds one or two of the warp's groups scanned while the others waited.
// Round 2 (faster, bit-identical results):
//   A  every lane evaluates LI_KNN_PB bricks per round and issues their hash probes back to back (first probe of the open-addressing
//      lookup split into issue / finish); found bricks go to the GROUP's list in shared memory through a group ballot;
//   B  the s-th listed brick of every group is scanned at the same time by group_scan_pipelined: the warp's trip count is the sum over
//      list slots of the longest slab in that slot, and the number of slots is the maximum over the groups of their found bricks --
//      instead of a sum over enumeration rounds.
// (Streaming the concatenated slabs through one cursor per group -- no per-brick restart at all -- was measured too and lost to the cursor
// arithmetic.)
#ifndef LI_KNN_PB
#define LI_KNN_PB 2          // bricks evaluated (hash probes in flight) per lane and round; 1 was slower, 3 no faster on H100
#endif
#ifndef LI_KNN_LIST
#define LI_KNN_LIST 32       // found bricks a group lists before it scans them ...
#endif
// ... and never fewer than one round can find: LI_KNN_PB * G bricks are probed between two looks at the fill level (G = 32: 64)
#define LI_KNN_LISTG(G) ((LI_KNN_LIST) > (LI_KNN_PB) * (G) ? (LI_KNN_LIST) : (LI_KNN_PB) * (G))
#ifndef LI_KNN_PREFETCH
#define LI_KNN_PREFETCH 4    // 128-byte lines of a found slab prefetched to L2 when it is listed (helps with a cold L2)
#endif
__device__ __forceinline__ uint4 li_brick_probe_issue(const uint4* __restrict__ ent, unsigned mask, unsigned long long key, unsigned& h) {
    h = li_hash(key) & mask;
    return __ldg(&ent[h]);
}
__device__ __forceinline__ bool li_brick_probe_finish(const uint4* __restrict__ ent, unsigned mask, unsigned long long key, unsigned h, uint4 e,
                                                      unsigned& first, unsigned& count) {
    for (unsigned i = 0; i <= mask; i++) {
        const unsigned long long k = (unsigned long long)e.x | ((unsigned long long)e.y << 32);
        if (k == key) { first = e.z; count = e.w; return true; }
        if (k == LI_EMPTY_KEY) return false;
        h = (h + 1) & mask;
        e = __ldg(&ent[h]);
    }
    return false;
}
template <int G>
__device__ __forceinline__ void group_scan_listed(const float4* __restrict__ pool, const uint2* __restrict__ glist, int nl, float qx, float qy, float qz,
                                                  float thr, float (&ld)[5], int (&li)[5], int gl) {
    for (int s = 0; __any_sync(LI_FULL, s < nl); s++) {
        unsigned f = 0, c = 0;
        if (s < nl) {
            const uint2 e = glist[s];
            f = e.x;
            c = e.y;
        }
        group_scan_pipelined<G>(pool, f, c, qx, qy, qz, thr, ld, li, gl);
    }
}
// Exact 5-NN of Q = 32/G queries by one warp in lockstep. ALL 32 lanes must call; `valid` is group-uniform.
// gd/gi: ascending distances / pool offsets (-1 = missing), uniform within each group.
//
// Shell iteration on the brick-box distance dbox (a conservative lower bound of the distance from the query to any
// point stored in the brick):
//     invariant: every brick with dbox < lo2 has been scanned
//     step:      scan the bricks with lo2 <= dbox < hi2 (enumerated over the bounding box of the ball of radius sqrt(hi2)),
//                merge -> (n, g5);  stop if n == 5 and g5 <= hi2 (no unscanned brick can hold a closer point) or hi2 >= 5;
//                otherwise lo2 = hi2 and hi2 = g5 if 5 are known (one closing step) else 4*hi2 (sparse neighbourhood).
// The first shell is a guess (rho = seed radius): with a dense map most queries finish in it, the rest need one closing step.
// thr0: a bound already known for the 5th best (only candidates below it can matter) -- INFINITY unless an earlier stage
// (the cell-directory first round of the hybrid search, cells.cuh) handed it over.
// glist: this GROUP's list of found bricks (LI_KNN_LISTG(G) entries of shared memory).
template <int G>
__device__ __forceinline__ void knn5_lockstep(const MapDev& M, float rho2, bool valid, float qx, float qy, float qz, float (&gd)[5],
                                               int (&gi)[5], int gl, int gbase, uint2* __restrict__ glist, float thr0 = INFINITY) {
    constexpr int PB = LI_KNN_PB;
    constexpr int LIST = LI_KNN_LISTG(G);
    float ld[5];
    int li[5];
#pragma unroll
    for (int i = 0; i < 5; i++) {
        ld[i] = INFINITY;
        li[i] = -1;
        gd[i] = INFINITY;
        gi[i] = -1;
    }
    KnnGeom g;
    g.bs = M.bshift;
    g.ds = M.ds;
    const int bc = 1 << g.bs;
    const float B = (float)bc * g.ds;
    const float lim = (float)(LI_CELL_LIMIT - 16 * bc) * g.ds;
    const bool act = valid && isfinite(qx) && isfinite(qy) && isfinite(qz) && fabsf(qx) < lim && fabsf(qy) < lim && fabsf(qz) < lim;
    if (!act) {
        qx = 0.f; qy = 0.f; qz = 0.f;
    }
    g.margin = 1e-6f * (fabsf(qx) + fabsf(qy) + fabsf(qz) + 16.0f * B);
    const float inv_ds = 1.0f / g.ds;
    const float slk = 0.02f + 4e-7f * (fabsf(qx) + fabsf(qy) + fabsf(qz)) * inv_ds;
    const unsigned ltg = (1u << gl) - 1u;
    bool done = !act;
    float lo2 = 0.f, hi2 = rho2;
    while (__any_sync(LI_FULL, !done)) {
        const bool need = !done;
        const bool last = hi2 >= 5.0f;
        const float r = sqrtf(fminf(hi2, 5.0f)) * (1.0f + 1e-6f) + g.margin;
        const int lx = (int)floorf((qx - r) * inv_ds - slk) >> g.bs, hx = (int)floorf((qx + r) * inv_ds + slk) >> g.bs;
        const int ly = (int)floorf((qy - r) * inv_ds - slk) >> g.bs, hy = (int)floorf((qy + r) * inv_ds + slk) >> g.bs;
        const int lz = (int)floorf((qz - r) * inv_ds - slk) >> g.bs, hz = (int)floorf((qz + r) * inv_ds + slk) >> g.bs;
        const int nx = hx - lx + 1, ny = hy - ly + 1, nz = hz - lz + 1;
        const int nxy = nx * ny;
        const int total = need ? nxy * nz : 0;
        const float inv_nxy = 1.0f / (float)nxy, inv_nx = 1.0f / (float)nx;
        const float thr = (gi[4] >= 0) ? gd[4] : thr0;
        int nl = 0;
        for (int base = 0; __any_sync(LI_FULL, base < total); base += PB * G) {
            unsigned long long key[PB];
            unsigned hs[PB];
            uint4 ent[PB];
            bool want[PB];
#pragma unroll
            for (int k = 0; k < PB; k++) {
                const int idx = base + k * G + gl;
                want[k] = idx < total;
                const int iz = (int)(((float)idx + 0.5f) * inv_nxy);
                const int rem = idx - iz * nxy;
                const int iy = (int)(((float)rem + 0.5f) * inv_nx);
                const int ix = rem - iy * nx;
                const int kx = lx + ix, ky = ly + iy, kz = lz + iz;
                key[k] = 0ull;
                hs[k] = 0u;
                ent[k] = make_uint4(0u, 0u, 0u, 0u);
                if (want[k]) {
                    const int bs = g.bs;
                    // (brick coordinate -> first cell: the shift is done on the unsigned image, a negative int may not be shifted before C++20)
                    const float lox = (float)li_shl(kx, bs) * g.ds - g.margin, hix = (float)li_shl(kx + 1, bs) * g.ds + g.margin;
                    const float loy = (float)li_shl(ky, bs) * g.ds - g.margin, hiy = (float)li_shl(ky + 1, bs) * g.ds + g.margin;
                    const float loz = (float)li_shl(kz, bs) * g.ds - g.margin, hiz = (float)li_shl(kz + 1, bs) * g.ds + g.margin;
                    const float ex = fmaxf(0.f, fmaxf(lox - qx, qx - hix));
                    const float ey = fmaxf(0.f, fmaxf(loy - qy, qy - hiy));
                    const float ez = fmaxf(0.f, fmaxf(loz - qz, qz - hiz));
                    const float dbox = (ex * ex + ey * ey + ez * ez) * (1.0f - 1e-6f);
                    const bool in_shell = dbox >= lo2 && (last ? dbox <= 5.0f : dbox < hi2);
                    want[k] = in_shell && dbox < thr;
                    if (want[k]) {
                        key[k] = li_pack_key(kx, ky, kz);
                        ent[k] = li_brick_probe_issue(M.ent, M.mask, key[k], hs[k]);
                    }
                }
            }
#pragma unroll
            for (int k = 0; k < PB; k++) {
                unsigned first = 0, count = 0;
                bool found = false;
                if (want[k]) {
                    found = li_brick_probe_finish(M.ent, M.mask, key[k], hs[k], ent[k], first, count);
                    found = found && count > 0u;
                }
                const unsigned fm = grp_ballot<G>(found, gbase);
                LI_EMUL_ASSERT(nl + __popc(fm) <= LIST);
                if (found) glist[nl + __popc(fm & ltg)] = make_uint2(first, count);
                nl += __popc(fm);
#if LI_KNN_PREFETCH && !defined(LI_SIMT_EMUL)
                // the slab will be read by the whole group a few hundred cycles from now: start moving its first lines towards L2
                if (found) {
                    const char* pf = reinterpret_cast<const char*>(M.pool + first);
                    const unsigned bytes = count * 16u;
#pragma unroll
                    for (int l = 0; l < LI_KNN_PREFETCH; l++)
                        if ((unsigned)l * 128u < bytes) asm volatile("prefetch.global.L2 [%0];" ::"l"(pf + l * 128));
                }
#endif
            }
            if (__any_sync(LI_FULL, nl > LIST - PB * G)) {   // the next round could find PB * G more
                __syncwarp();
                group_scan_listed<G>(M.pool, glist, nl, qx, qy, qz, thr, ld, li, gl);
                nl = 0;
                __syncwarp();
            }
        }
        __syncwarp();
        group_scan_listed<G>(M.pool, glist, nl, qx, qy, qz, thr, ld, li, gl);
        __syncwarp();
        group_merge<G>(ld, li, gd, gi, gl, gbase);
        if (need) {
            const bool full = gi[4] >= 0;
            if (last || (full && gd[4] <= hi2)) {
                done = true;
            } else {
                lo2 = hi2;
                hi2 = full ? fminf(gd[4] * (1.0f + 1e-6f), 5.0f) : fminf(4.0f * hi2, 5.0f);
                if (full && hi2 >= 5.0f) hi2 = 5.0f;
            }
        }
    }
}
#define LI_KNN_SMEM_DECL(G, W) __shared__ uint2 s_glist[W][32 / (G)][LI_KNN_LISTG(G)]
#define LI_KNN_CALL(G, M, rho2, valid, QX_, QY_, QZ_, gd, gi, gl, gbase, THR0_) \
    knn5_lockstep<G>(M, rho2, valid, QX_, QY_, QZ_, gd, gi, gl, gbase, s_glist[threadIdx.x >> 5][(threadIdx.x & 31) / (G)], THR0_)

// ---- search kernel of an ICP pass: world transform + 5-NN for every scan point -----------------------
// HOST = true: the scan has not been copied yet -- `raw` is a device-visible alias of the caller's page-locked host
// buffer (liinit_scan_attach_host) and the kernel pulls the coordinates over PCIe itself (one contiguous
// Q*stride*4-byte read per warp batch, hidden behind the other warps' searches), leaving the packed copy in
// S.body for the plane kernel and the later passes. No staging copy, no repack launch in front of the search.
// SEEDED = true (a separate instantiation, so that the first-pass kernel keeps its registers): see below.
template <int G, bool HOST, bool SEEDED = false>
__global__ void __launch_bounds__(LI_KNN_THREADS, LI_KNN_MIN_BLOCKS)
k_knn_scan(MapDev M, ScanDev S, PoseD P, float rho2, const float* __restrict__ raw, int stride) {
    constexpr int Q = Grp<G>::Q;
    LI_KNN_SMEM_DECL(G, LI_KNN_THREADS / 32);
    const int lane = threadIdx.x & 31;
    const int gl = lane % G, gid = lane / G, gbase = gid * G;
    const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int nwarps = (gridDim.x * blockDim.x) >> 5;
    for (int qb = warp_global * Q; qb < S.n; qb += nwarps * Q) {   // warp-uniform
        const int q = qb + gid;
        const bool valid = q < S.n;
        float wx = 0.f, wy = 0.f, wz = 0.f;
        if (HOST) {
            float bx = 0.f, by = 0.f, bz = 0.f;
            if (G >= 4) {   // lanes 0..2 of the group fetch x, y, z: the warp's addresses are contiguous for stride 3
                float v = 0.f;
                if (valid && gl < 3) v = raw[(size_t)q * stride + gl];
                bx = __shfl_sync(LI_FULL, v, gbase);
                by = __shfl_sync(LI_FULL, v, gbase + 1);
                bz = __shfl_sync(LI_FULL, v, gbase + 2);
            } else if (valid) {
                const float* s = raw + (size_t)q * stride;
                bx = s[0]; by = s[1]; bz = s[2];
            }
            if (valid) {
                if (gl == 0) S.body[q] = make_float4(bx, by, bz, 0.f);
                li_body_to_world(P, bx, by, bz, wx, wy, wz);
            }
        } else if (valid) {
            float4 b = __ldg(&S.body[q]);
            li_body_to_world(P, b.x, b.y, b.z, wx, wy, wz);
        }
        // A later search pass of the same scan (laserMapping.cpp:1102-1106: rematch after convergence) starts from what the previous one
        // found: the five stored neighbours still exist in the map (the host only sets `seeded` while no point has been removed since), so
        // the 5th-neighbour distance at the moved query cannot exceed the largest of THEIR distances from it. That bound is the radius of
        // the first -- and then only -- shell and the candidate threshold: one shell, a handful of inserts. Exactness is untouched.
        float rho2q = rho2, thr0 = INFINITY;
        if (SEEDED) {
            float bmax = 0.f;
            bool miss = false;
#pragma unroll
            for (int k = 0; k < 5; k++) {
                if (k % G == gl && valid) {
                    const float4 e = S.near_xyz[(size_t)q * 5 + k];
                    if (e.w == 0.f) miss = true;
                    else bmax = fmaxf(bmax, li_dist2(wx, wy, wz, e.x, e.y, e.z));
                }
            }
#pragma unroll
            for (int o = (G > 4 ? 4 : G / 2); o >= 1; o >>= 1) bmax = fmaxf(bmax, __shfl_xor_sync(LI_FULL, bmax, o));   // ranks live in lanes 0..min(G,5)-1 (+ wrap for G < 5)
            if (G > 4) bmax = __shfl_sync(LI_FULL, bmax, gbase);
            const bool any_miss = grp_ballot<G>(miss, gbase) != 0u;
            if (valid && !any_miss && bmax < 5.0f) {
                rho2q = bmax * (1.0f + 2e-6f) + 1e-12f;
                thr0 = __uint_as_float(__float_as_uint(bmax) + 1u);   // smallest float above the bound: d <= bmax passes `d < thr0`
            }
        }
        float gd[5];
        int gi[5];
        LI_KNN_CALL(G, M, rho2q, valid, wx, wy, wz, gd, gi, gl, gbase, thr0);
        if (valid) {
            if (gl == 0) S.world[q] = make_float4(wx, wy, wz, 0.f);
            // Nearest_Points as COPIES (ScanDev::near_xyz; w = 1 found, 0 missing rank): the group's lanes share the five gathers --
            // the slabs were read a moment ago, these are cache hits -- and the plane kernel of this pass needs no pool offsets
#pragma unroll
            for (int k = 0; k < 5; k++) {
                if (k % G == gl) {
                    float4 e = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (gi[k] >= 0) {
                        e = __ldg(&M.pool[gi[k]]);
                        e.w = 1.0f;
                    }
                    S.near_xyz[(size_t)q * 5 + k] = e;
                }
            }
        }
    }
}

// ---- stand-alone Nearest_Search for arbitrary world-frame queries --------------------------------------
template <int G>
__global__ void __launch_bounds__(256) k_knn_queries(MapDev M, const float4* __restrict__ qpts, int n, int* __restrict__ ids,
                                                     float* __restrict__ d2, float rho2) {
    constexpr int Q = Grp<G>::Q;
    LI_KNN_SMEM_DECL(G, 256 / 32);
    const int lane = threadIdx.x & 31;
    const int gl = lane % G, gid = lane / G, gbase = gid * G;
    const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int nwarps = (gridDim.x * blockDim.x) >> 5;
    for (int qb = warp_global * Q; qb < n; qb += nwarps * Q) {
        const int q = qb + gid;
        const bool valid = q < n;
        float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
        if (valid) p = __ldg(&qpts[q]);
        float gd[5];
        int gi[5];
        LI_KNN_CALL(G, M, rho2, valid, p.x, p.y, p.z, gd, gi, gl, gbase, INFINITY);
        if (valid && gl == 0) {
#pragma unroll
            for (int k = 0; k < 5; k++) {
                ids[(size_t)q * 5 + k] = gi[k];
                d2[(size_t)q * 5 + k] = (gi[k] >= 0) ? gd[k] : -1.f;
            }
        }
    }
}
