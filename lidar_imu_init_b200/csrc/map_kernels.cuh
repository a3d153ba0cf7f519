// map_kernels.cuh -- device-resident map: build / insert / downsample-insert.
//
// Replaces KD_TREE::Build (ikd_Tree.cpp:336-347), KD_TREE::Add_Points (ikd_Tree.cpp:381-456) and the
// classification of map_incremental (laserMapping.cpp:516-559). All batch semantics are derived in
// DESIGN.md section 4: after Add_Points(batch, downsample_on=true) every voxel hit by the batch holds exactly the
// point closest to the voxel centre among {its live points} U {the batch's points in it} (new beats
// existing on ties, later beats earlier among new), which is what the reference's sequential loop
// produces, independent of order.
#pragma once
#include "common.cuh"
#include "cells.cuh"   // li_sb_mark: super-brick occupancy of the cell-directory search (no-op unless enabled)

// ---- staging: strided host layout -> float4 -------------------------------------------------------
__global__ void k_repack(const float* __restrict__ src, int stride, int n, float4* __restrict__ dst) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* s = src + (size_t)i * stride;
    dst[i] = make_float4(s[0], s[1], s[2], 0.f);
}

// same, keeping one more float (a per-point time stamp, e.g. PointType.curvature) in w; attr (optional, PointType layout only):
// {normal_x, normal_y, normal_z, intensity} = floats 4-6 and 8
__global__ void k_repack_t(const float* __restrict__ src, int stride, int tidx, int n, float4* __restrict__ dst, float4* __restrict__ attr) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* s = src + (size_t)i * stride;
    dst[i] = make_float4(s[0], s[1], s[2], tidx >= 0 ? s[tidx] : 0.f);
    if (attr) attr[i] = make_float4(s[4], s[5], s[6], s[8]);
}

__global__ void k_map_clear(uint4* ent, uint4* aux, unsigned slots) {
    unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= slots) return;
    ent[i] = make_uint4(0xffffffffu, 0xffffffffu, 0u, 0u);
    aux[i] = make_uint4(0u, 0u, 0u, 0u);
}

__device__ __forceinline__ bool li_point_cells(const MapDev& M, float4 p, int& cx, int& cy, int& cz) {
    if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z))) return false;
    float lim = (float)(LI_CELL_LIMIT - 2) * M.ds;
    if (fabsf(p.x) >= lim || fabsf(p.y) >= lim || fabsf(p.z) >= lim) return false;
    cx = li_cell(p.x, M.ds);
    cy = li_cell(p.y, M.ds);
    cz = li_cell(p.z, M.ds);
    return true;
}

__device__ __forceinline__ unsigned li_voxel_in_brick(const MapDev& M, int cx, int cy, int cz) {
    int m = (1 << M.bshift) - 1;
    return (unsigned)(((cx & m) << (2 * M.bshift)) | ((cy & m) << M.bshift) | (cz & m));
}


// Index of the downsample box that CONTAINS x as the reference tests membership (Search_by_range / Delete_by_range,
// ikd_Tree.cpp:633,980): box k = [fl(k*ds), fl(fl(k*ds)+ds)). It equals the division index c = floor(fl(x/ds)) except
// within one ulp of a box edge, where x can sit in box c-1 / c+1 or in NO box (the float boxes leave one-ulp gaps).
// Grid-aligned synthetic scenes (walls at k*ds) hit this systematically, so it is reproduced exactly.
#define LI_NO_BOX 0xfffffffeu
__device__ __forceinline__ bool li_box_index(float x, float ds, int c, int& b) {
    float cf = (float)c;
    float mn = __fmul_rn(cf, ds), mx = __fadd_rn(mn, ds);
    if (x >= mn && x < mx) { b = c; return true; }
    if (x < mn) {
        float m1 = __fmul_rn(cf - 1.0f, ds), x1 = __fadd_rn(m1, ds);
        if (x >= m1 && x < x1) { b = c - 1; return true; }
    } else {
        float m1 = __fmul_rn(cf + 1.0f, ds), x1 = __fadd_rn(m1, ds);
        if (x >= m1 && x < x1) { b = c + 1; return true; }
    }
    b = c;
    return false;
}

// Where a map point is STORED: the brick of its box index (so that the box test of a later Add_Points finds it in
// the brick of that box) and its voxel-in-brick id, or LI_NO_BOX when it lies in no downsample box.
__device__ __forceinline__ void li_storage(const MapDev& M, float4 p, int cx, int cy, int cz, unsigned long long& brick_key, unsigned& vib) {
    int bx, by, bz;
    bool ok = li_box_index(p.x, M.ds, cx, bx);
    ok = li_box_index(p.y, M.ds, cy, by) && ok;
    ok = li_box_index(p.z, M.ds, cz, bz) && ok;
    if (ok) {
        brick_key = li_pack_key(bx >> M.bshift, by >> M.bshift, bz >> M.bshift);
        vib = li_voxel_in_brick(M, bx, by, bz);
    } else {
        brick_key = li_pack_key(cx >> M.bshift, cy >> M.bshift, cz >> M.bshift);
        vib = LI_NO_BOX;
    }
}

// add a hash slot to the batch's touched list exactly once (aux.w is the membership flag)
__device__ __forceinline__ void li_touch(const MapDev& M, int s) {
    if (atomicExch(&M.aux[s].w, 1u) == 0u) {
        const int t = atomicAdd(&M.counters[CNT_TOUCHED], 1);
        LI_EMUL_ASSERT(t >= 0 && (unsigned)t <= M.mask);   // every hash slot is listed at most once per batch
        M.touched_list[t] = s;
    }
}

// ---- plain insert (Build, Add_Points(.., false)) -------------------------------------------------
// pass 1: find-or-create the brick of every point, count pending points per brick.
__global__ void k_ins_count(MapDev M, const float4* __restrict__ pts, int n, const int* __restrict__ sel, int want,
                            int* __restrict__ slot_of) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    slot_of[i] = -1;
    if (sel && sel[i] != want) return;
    int cx, cy, cz;
    float4 p = pts[i];
    if (!li_point_cells(M, p, cx, cy, cz)) {
        atomicAdd(&M.counters[CNT_DROPPED], 1);
        return;
    }
    unsigned long long key;
    unsigned vib;
    li_storage(M, p, cx, cy, cz, key, vib);
    bool created = false;
    int s = li_brick_find_or_insert(M.ent, M.mask, key, &created);
    if (s < 0) {
        atomicOr(&M.counters[CNT_ERR], ERR_HASH_FULL);
        return;
    }
    slot_of[i] = s;
    if (created) {
        const int nb = atomicAdd(&M.counters[CNT_BRICKS], 1);
        LI_EMUL_ASSERT(nb >= 0 && (unsigned)nb <= M.mask);
        M.brick_slots[nb] = s;
        li_sb_mark(M, key);
    }
    atomicAdd(&M.aux[s].y, 1u);
    li_touch(M, s);
}

// pass 2: one warp per touched brick -- grow its slab when count + pending exceeds the capacity.
__global__ void k_ins_reserve(MapDev M) {
    const int lane = threadIdx.x & 31;
    const int nw = (gridDim.x * blockDim.x) >> 5, ntouched = M.counters[CNT_TOUCHED];
    for (int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < ntouched; w += nw) {   // fixed grid, the count lives on the device
    int s = M.touched_list[w];
    uint4 e = M.ent[s];
    uint4 a = M.aux[s];
    unsigned need = e.w + a.y;
    if (need > a.x) {
        unsigned ncap = need + (need >> 1);
        if (ncap < 16u) ncap = 16u;
        ncap = (ncap + 7u) & ~7u;
        unsigned long long off = 0;
        if (lane == 0) off = atomicAdd(M.pool_top, (unsigned long long)ncap);
        off = __shfl_sync(LI_FULL, off, 0);
        if (off + ncap > M.pool_cap) {
            if (lane == 0) {
                atomicOr(&M.counters[CNT_ERR], ERR_POOL_FULL);
                M.aux[s].y = 0u;   // nothing will be appended to this brick
                // pool_top is NOT rolled back here: between this warp's add and a subtraction other warps reserve, and one of them may fit
                // and keep a slab ABOVE the value the subtractions end on -- the next reservation would be handed the same slots. The
                // allocator stays beyond the capacity for the rest of the call (every later reservation of this batch fails, the call
                // returns LIINIT_ERR_CAPACITY), and the host then has k_pool_top_recompute put it back on the end of the last slab in use.
            }
            continue;
        }
        for (unsigned j = lane; j < e.w; j += 32) M.pool[off + j] = M.pool[e.z + j];
        if (lane == 0) {
            M.ent[s].z = (unsigned)off;
            M.aux[s].x = ncap;
        }
    }
    if (lane == 0) M.aux[s].z = 0u;
    }
}

// After a failed reservation (host side, check_map_err): pool_top := end of the highest slab any brick owns (pool_top zeroed first).
__global__ void k_pool_top_recompute(MapDev M, int nbricks) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nbricks) return;
    const int s = M.brick_slots[i];
    const unsigned cap = M.aux[s].x;
    if (cap) atomicMax(M.pool_top, (unsigned long long)M.ent[s].z + cap);
}

// pass 3: append. ent.count is not modified until the commit, so first+count is the append base.
__global__ void k_ins_append(MapDev M, const float4* __restrict__ pts, int n, const int* __restrict__ slot_of) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int s = slot_of[i];
    if (s < 0) return;
    uint4 e = M.ent[s];
    uint4 a = M.aux[s];
    if (a.y == 0u) return;   // reservation failed
    unsigned j = atomicAdd(&M.aux[s].z, 1u);
    float4 p = pts[i];
    int cx = li_cell(p.x, M.ds), cy = li_cell(p.y, M.ds), cz = li_cell(p.z, M.ds);
    unsigned long long key;
    unsigned vib;
    li_storage(M, p, cx, cy, cz, key, vib);
    p.w = __uint_as_float(vib);
    LI_EMUL_ASSERT(e.w + j < a.x && (unsigned long long)e.z + a.x <= M.pool_cap);   // inside the brick's slab, the slab inside the pool
    M.pool[(size_t)e.z + e.w + j] = p;
}

// pass 4: commit counts.
__global__ void k_ins_commit(MapDev M) {
    const int nt = gridDim.x * blockDim.x, ntouched = M.counters[CNT_TOUCHED];
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < ntouched; t += nt) {
        int s = M.touched_list[t];
        unsigned f = M.aux[s].z;
        M.ent[s].w += f;
        M.aux[s].y = 0u;
        M.aux[s].z = 0u;
        M.aux[s].w = 0u;
        atomicAdd(&M.counters[CNT_LIVE], (int)f);
    }
}

// ---- downsample insert (Add_Points(.., true)) --------------------------------------------------
// The reference walks the batch sequentially (ikd_Tree.cpp:388-426). For one downsample box the walk reduces to a
// tiny state machine over the box's current content E (count, best distance to the box centre, best point):
//   new point p (distance d_p):  p wins  <=>  !(E non-empty && d_best < d_p)      (strict '<': new wins ties)
//   if |E| > 1 or p wins or same_point(p, best):   box is deleted, the winner is (re)inserted, E := {winner}
// with two float-box subtleties that matter on grid-aligned data: a new point can lie OUTSIDE its own box (ulp edge:
// then it is inserted but never seen by later box queries, E := {} after it wins), and an existing point belongs to
// the box that CONTAINS it (li_box_index), not to the cell of its division index.
// Boxes are independent of each other, so: one thread per box replays ITS new points in batch order.
struct VoxTmp {
    unsigned long long* keys;   // box key (division cell of the new points)
    int* head;                  // newest batch index linked into this box (-1 = none)
    unsigned mask;
    // Add_Points(downsample) only (nullptr for the scan voxel grid, which shares the hash):
    int* coupled;               // 1: the box shares a point with another box that also receives new points -> replayed by k_ds_coupled
    int4* sum;                  // what k_ds_scan found in the box: {count, best distance (float bits), pool offset of the best point, any brick}
    int* clist;                 // slots of the coupled boxes [counters[CNT_COUPLED]]
};

__global__ void k_vox_clear(VoxTmp V) {
    unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > V.mask) return;
    V.keys[i] = LI_EMPTY_KEY;
    V.head[i] = -1;
    if (V.coupled) V.coupled[i] = 0;
}

// Distance of p to the centre of its downsample box, float arithmetic of ikd_Tree.cpp:389-401.
__device__ __forceinline__ float li_center_dist_cell(float qx, float qy, float qz, int cx, int cy, int cz, float ds) {
    float mnx = __fmul_rn((float)cx, ds), mxx = __fadd_rn(mnx, ds);
    float mny = __fmul_rn((float)cy, ds), mxy = __fadd_rn(mny, ds);
    float mnz = __fmul_rn((float)cz, ds), mxz = __fadd_rn(mnz, ds);
    float mx = (float)__dadd_rn((double)mnx, __ddiv_rn((double)__fsub_rn(mxx, mnx), 2.0));
    float my = (float)__dadd_rn((double)mny, __ddiv_rn((double)__fsub_rn(mxy, mny), 2.0));
    float mz = (float)__dadd_rn((double)mnz, __ddiv_rn((double)__fsub_rn(mxz, mnz), 2.0));
    return li_dist2(qx, qy, qz, mx, my, mz);
}

// pass D1: link every selected new point into the list of its box; reserve one slot in the brick it would be stored in.
__global__ void k_ds_link(MapDev M, VoxTmp V, const float4* __restrict__ pts, int n, const int* __restrict__ sel, int want,
                          int* __restrict__ next_of, int* __restrict__ slot_of, int* __restrict__ ins) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    next_of[i] = -2;   // not part of the batch
    slot_of[i] = -1;
    ins[i] = 0;
    if (sel && sel[i] != want) return;
    int cx, cy, cz;
    float4 p = pts[i];
    if (!li_point_cells(M, p, cx, cy, cz)) {
        atomicAdd(&M.counters[CNT_DROPPED], 1);
        return;
    }
    // storage brick: worst case every new point is inserted
    unsigned long long skey;
    unsigned svib;
    li_storage(M, p, cx, cy, cz, skey, svib);
    bool created = false;
    int s = li_brick_find_or_insert(M.ent, M.mask, skey, &created);
    if (s < 0) {
        atomicOr(&M.counters[CNT_ERR], ERR_HASH_FULL);
        return;
    }
    if (created) {
        const int nb = atomicAdd(&M.counters[CNT_BRICKS], 1);
        LI_EMUL_ASSERT(nb >= 0 && (unsigned)nb <= M.mask);
        M.brick_slots[nb] = s;
        li_sb_mark(M, skey);
    }
    slot_of[i] = s;
    atomicAdd(&M.aux[s].y, 1u);
    li_touch(M, s);
    // box list
    unsigned long long key = li_pack_key(cx, cy, cz);
    unsigned h = li_hash(key) & V.mask;
    int slot = -1;
    for (unsigned t = 0; t <= V.mask; t++) {
        unsigned long long k = *reinterpret_cast<volatile unsigned long long*>(&V.keys[h]);
        if (k == key) { slot = (int)h; break; }
        if (k == LI_EMPTY_KEY) {
            unsigned long long old = atomicCAS(&V.keys[h], LI_EMPTY_KEY, key);
            if (old == LI_EMPTY_KEY || old == key) { slot = (int)h; break; }
        }
        h = (h + 1) & V.mask;
    }
    if (slot < 0) {
        atomicOr(&M.counters[CNT_ERR], ERR_HASH_FULL);
        return;
    }
    next_of[i] = atomicExch(&V.head[slot], i);
}

struct DsBox {
    float mn[3], mx[3];
    float mx_prev[3], mn_next[3];   // upper end of the box below / lower end of the box above, per axis
    int c[3];                       // division cell
    int blo[3], bhi[3];             // range of brick coordinates per axis that can store a point of this box
};
__device__ __forceinline__ bool li_in_box(const DsBox& B, const float4& q) {
    return q.x >= B.mn[0] && q.x < B.mx[0] && q.y >= B.mn[1] && q.y < B.mx[1] && q.z >= B.mn[2] && q.z < B.mx[2];
}
__device__ __forceinline__ void li_ds_box(const MapDev& M, const float4& ph, DsBox& B) {
    B.c[0] = li_cell(ph.x, M.ds); B.c[1] = li_cell(ph.y, M.ds); B.c[2] = li_cell(ph.z, M.ds);
    const int bm = (1 << M.bshift) - 1;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        const float cf = (float)B.c[a];
        B.mn[a] = __fmul_rn(cf, M.ds);
        B.mx[a] = __fadd_rn(B.mn[a], M.ds);
        B.mx_prev[a] = __fadd_rn(__fmul_rn(cf - 1.0f, M.ds), M.ds);
        B.mn_next[a] = __fmul_rn(cf + 1.0f, M.ds);
        const int b0 = B.c[a] >> M.bshift;
        B.blo[a] = (B.mn[a] < B.mx_prev[a] && (B.c[a] & bm) == 0) ? b0 - 1 : b0;      // overlap with box c-1, which lives in the brick below
        B.bhi[a] = (B.mx[a] > B.mn_next[a] && (B.c[a] & bm) == bm) ? b0 + 1 : b0;     // overlap with box c+1, which lives in the brick above
    }
}
// slot of a box in the batch's temporary hash, -1 when the batch has no new point for that cell
__device__ __forceinline__ int li_vox_find(const VoxTmp& V, unsigned long long key) {
    unsigned h = li_hash(key) & V.mask;
    for (unsigned t = 0; t <= V.mask; t++) {
        const unsigned long long k = V.keys[h];
        if (k == key) return V.head[h] >= 0 ? (int)h : -1;
        if (k == LI_EMPTY_KEY) return -1;
        h = (h + 1) & V.mask;
    }
    return -1;
}
__device__ __forceinline__ void li_couple(const MapDev& M, const VoxTmp& V, int v) {
    if (atomicExch(&V.coupled[v], 1) == 0) V.clist[atomicAdd(&M.counters[CNT_COUPLED], 1)] = v;
}
// x lies in box B.c (or is a new point filed under it). Per axis lo[a]..hi[a] is the range of cell offsets (-1, 0, +1) whose float
// interval contains x[a] (empty when lo > hi: a one-ulp gap). Every OTHER box that contains x and receives new points in this batch is
// coupled with box v: the reference's sequential walk lets such boxes see each other's deletions and insertions.
__device__ __forceinline__ void li_couple_neighbours(const MapDev& M, const VoxTmp& V, const DsBox& B, int v, const int (&lo)[3], const int (&hi)[3]) {
    for (int oz = lo[2]; oz <= hi[2]; oz++)
        for (int oy = lo[1]; oy <= hi[1]; oy++)
            for (int ox = lo[0]; ox <= hi[0]; ox++) {
                if ((ox | oy | oz) == 0) continue;
                const int w = li_vox_find(V, li_pack_key(B.c[0] + ox, B.c[1] + oy, B.c[2] + oz));
                if (w >= 0) {
                    li_couple(M, V, v);
                    li_couple(M, V, w);
                }
            }
}

// pass D3a: one thread per box -- what the box holds before the batch (count, the point closest to the box centre: first minimum in
// visiting order), and which boxes are COUPLED. The float boxes of neighbouring cells overlap by one ulp here and there; a point inside
// an overlap belongs to two boxes. When both receive new points in one batch the reference's walk is order dependent ACROSS the boxes
// (the first one may delete the shared point before the second one looks), so such boxes -- through a shared existing point or through
// a new point that lies in the other box -- are taken out of the parallel replay and walked in batch order by k_ds_coupled.
// (Found by tools/emul_fuzz.py on lattice clouds 5 km from the origin: one changed-box count off by one, same live set.)
__global__ void k_ds_scan(MapDev M, VoxTmp V, const float4* __restrict__ pts, const int* __restrict__ next_of) {
    unsigned v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v > V.mask) return;
    const int head = V.head[v];
    if (head < 0) return;
    DsBox B;
    li_ds_box(M, pts[head], B);
    int nE = 0;
    float bd = INFINITY;
    int bref = -1;
    bool have = false;
    for (int kz = B.blo[2]; kz <= B.bhi[2]; kz++)
        for (int ky = B.blo[1]; ky <= B.bhi[1]; ky++)
            for (int kx = B.blo[0]; kx <= B.bhi[0]; kx++) {
                unsigned first = 0, count = 0;
                // (li_brick_find uses the read-only path; ent is not modified between D2's reserve and this kernel)
                if (!li_brick_find(M.ent, M.mask, li_pack_key(kx, ky, kz), first, count)) continue;
                have = true;
                for (unsigned j = 0; j < count; j++) {
                    const float4 q = M.pool[(size_t)first + j];
                    if (__float_as_uint(q.w) == 0xffffffffu || !li_in_box(B, q)) continue;
                    nE++;
                    const float d = li_center_dist_cell(q.x, q.y, q.z, B.c[0], B.c[1], B.c[2], M.ds);
                    if (d < bd) { bd = d; bref = (int)(first + j); }
                    const float qa[3] = {q.x, q.y, q.z};
                    int lo[3], hi[3];
                    bool shared = false;
#pragma unroll
                    for (int a = 0; a < 3; a++) {
                        lo[a] = qa[a] < B.mx_prev[a] ? -1 : 0;
                        hi[a] = qa[a] >= B.mn_next[a] ? 1 : 0;
                        shared = shared || lo[a] != 0 || hi[a] != 0;
                    }
                    if (shared) li_couple_neighbours(M, V, B, (int)v, lo, hi);
                }
            }
    // new points filed under this cell that lie in another box too (or only there)
    for (int t = head; t >= 0; t = next_of[t]) {
        const float4 p = pts[t];
        const float pa[3] = {p.x, p.y, p.z};
        int lo[3], hi[3];
        bool plain = true;
#pragma unroll
        for (int a = 0; a < 3; a++) {
            const float cf = (float)B.c[a];
            const float mn_prev = __fmul_rn(cf - 1.0f, M.ds), mx_next = __fadd_rn(B.mn_next[a], M.ds);
            const bool in_prev = pa[a] >= mn_prev && pa[a] < B.mx_prev[a];
            const bool in_own = pa[a] >= B.mn[a] && pa[a] < B.mx[a];
            const bool in_next = pa[a] >= B.mn_next[a] && pa[a] < mx_next;
            lo[a] = in_prev ? -1 : (in_own ? 0 : (in_next ? 1 : 2));       // the intervals are consecutive: the offsets that hold form a range
            hi[a] = in_next ? 1 : (in_own ? 0 : (in_prev ? -1 : -2));      // (lo > hi: a one-ulp gap -- the point is in no box at all)
            plain = plain && lo[a] == 0 && hi[a] == 0;
        }
        if (!plain) li_couple_neighbours(M, V, B, (int)v, lo, hi);
    }
    V.sum[v] = make_int4(nE, __float_as_int(bd), bref, have ? 1 : 0);
}

// pass D3: one thread per box that is not coupled -- replay the box's new points in batch order (see the state machine above).
// Existing losers are tombstoned (w = 0xffffffff), ins[i] = 1 marks the new points that end up in the map.
//
// Which existing points are "in the box" is decided GEOMETRICALLY, as Search_by_range / Delete_by_range decide it
// (vertex_min <= x && x < vertex_max per axis, ikd_Tree.cpp:633,980), not by the voxel id a point was filed under: the float boxes
// [fl(k ds), fl(fl(k ds) + ds)) of neighbouring k do not tile the axis -- they leave one-ulp gaps AND one-ulp overlaps, and a
// point inside an overlap belongs to both boxes although it is stored under one index only (found by tools/emul_fuzz.py: lattice
// points 900 m from the origin). Such a point can sit in the adjacent brick when the box touches a brick face, so up to two bricks
// per axis are looked at -- one in all but ulp cases.
__global__ void k_ds_replay(MapDev M, VoxTmp V, const float4* __restrict__ pts, int* __restrict__ next_of,
                            int* __restrict__ ins) {
    unsigned v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v > V.mask) return;
    int head = V.head[v];
    if (head < 0) return;
    if (V.coupled[v]) return;   // k_ds_coupled walks it
    DsBox B;
    li_ds_box(M, pts[head], B);
    const int cx = B.c[0], cy = B.c[1], cz = B.c[2];
    // existing content of the box (k_ds_scan)
    const int4 sm = V.sum[v];
    int nE = sm.x;
    float bd = __int_as_float(sm.y);
    long long bref = sm.z;    // >= 0: pool offset of an existing point; <= -2: new point index -(bref+2)
    float bxx = 0, byy = 0, bzz = 0;
    if (bref >= 0) {
        const float4 q = M.pool[bref];
        bxx = q.x; byy = q.y; bzz = q.z;
    }
    const bool have = sm.w != 0;
    bool modified = false;
    int changed = 0;
    // batch order = ascending index. Short lists (the usual box: one to three new points): repeatedly take the smallest index greater than
    // the last one, no stores; long lists: the links are sorted once (merge sort), then replayed in one walk
    const bool sorted_walk = li_list_longer_than(head, next_of, LI_LIST_SELECT_MAX);
    if (sorted_walk) head = li_list_sort_ascending(head, next_of);
    int last = -1, walk = head;
    for (;;) {
        int cur;
        if (sorted_walk) {
            cur = walk;
            if (cur < 0) break;
            walk = next_of[cur];
        } else {
            cur = 0x7fffffff;
            for (int t = head; t >= 0; t = next_of[t])
                if (t > last && t < cur) cur = t;
            if (cur == 0x7fffffff) break;
            last = cur;
        }
        float4 p = pts[cur];
        float dp = li_center_dist_cell(p.x, p.y, p.z, cx, cy, cz, M.ds);
        bool newwins = !(nE > 0 && bd < dp);
        bool same = newwins || (nE > 0 && fabsf(__fsub_rn(p.x, bxx)) < 1e-6f && fabsf(__fsub_rn(p.y, byy)) < 1e-6f &&
                                fabsf(__fsub_rn(p.z, bzz)) < 1e-6f);   // same_point, EPSS (ikd_Tree.cpp:1269-1271)
        if (nE > 1 || same) {
            modified = true;
            changed++;
            if (newwins) {
                if (bref <= -2) ins[-(bref + 2)] = 0;   // an earlier in-box new point is deleted with the box
                ins[cur] = 1;
                if (li_in_box(B, p)) {
                    nE = 1; bd = dp; bref = -((long long)cur + 2); bxx = p.x; byy = p.y; bzz = p.z;
                } else {   // the new point lies outside its own box (ulp edge): inserted, but no later query of THIS box sees it
                    nE = 0; bd = INFINITY; bref = -1;
                }
            } else {
                nE = 1;   // the best point survives alone
            }
        }
    }
    if (changed) atomicAdd(&M.counters[CNT_CHANGED], changed);
    if (!(modified && have)) return;
    // the box was deleted at least once: every existing point in it except a surviving best one goes; the bricks that hold tombstones are
    // put on the touched list so that the compaction squeezes them out
    for (int kz = B.blo[2]; kz <= B.bhi[2]; kz++)
        for (int ky = B.blo[1]; ky <= B.bhi[1]; ky++)
            for (int kx = B.blo[0]; kx <= B.bhi[0]; kx++) {
                const unsigned long long key = li_pack_key(kx, ky, kz);
                unsigned first = 0, count = 0;
                if (!li_brick_find(M.ent, M.mask, key, first, count)) continue;
                bool any = false;
                for (unsigned j = 0; j < count; j++) {
                    float4* qp = &M.pool[(size_t)first + j];
                    if (__float_as_uint(qp->w) == 0xffffffffu || !li_in_box(B, *qp)) continue;
                    if (nE == 1 && bref == (long long)first + j) continue;
                    qp->w = __uint_as_float(0xffffffffu);
                    any = true;
                }
                if (!any) continue;
                unsigned h = li_hash(key) & M.mask;
                for (unsigned t = 0; t <= M.mask; t++) {
                    unsigned long long k = *reinterpret_cast<volatile unsigned long long*>(&M.ent[h]);
                    if (k == key) { li_touch(M, (int)h); break; }
                    if (k == LI_EMPTY_KEY) break;
                    h = (h + 1) & M.mask;
                }
            }
}

// pass D3c: the coupled boxes (k_ds_scan), by ONE warp: their new points are gathered, put in batch order and walked the way the
// reference walks a batch -- for every point the box is looked up afresh (existing points that are still alive + the new points
// accepted so far that lie in it, both geometrically), so what one box deletes or inserts is seen by the next. The lanes share the
// work inside a step. An ulp-rare path: a handful of points per batch on sensor data, thousands only on lattice-aligned synthetic clouds.
__global__ void k_ds_coupled(MapDev M, VoxTmp V, const float4* __restrict__ pts, const int* __restrict__ next_of, int* __restrict__ ins,
                             int* __restrict__ cidx, int* __restrict__ csorted) {
    const int nc = M.counters[CNT_COUPLED];
    if (nc == 0) return;
    const int lane = threadIdx.x & 31;
    __shared__ int s_n;
    if (lane == 0) s_n = 0;
    __syncwarp();
    for (int b = lane; b < nc; b += 32)
        for (int t = V.head[V.clist[b]]; t >= 0; t = next_of[t]) cidx[atomicAdd(&s_n, 1)] = t;
    __syncwarp();
    const int n = s_n;
    for (int a = lane; a < n; a += 32) {   // rank sort: the indices are distinct
        const int x = cidx[a];
        int r = 0;
        for (int b = 0; b < n; b++) r += cidx[b] < x;
        csorted[r] = x;
    }
    __syncwarp();
    // the walk itself: one point after the other, the warp shares the work INSIDE a step (lane-strided scans, a lexicographic minimum
    // over (distance, visiting order) so that "first minimum in visiting order" is what a single thread would have found)
    int changed = 0;
    for (int pos = 0; pos < n; pos++) {
        const int cur = csorted[pos];
        const float4 p = pts[cur];
        DsBox B;
        li_ds_box(M, p, B);
        const float dp = li_center_dist_cell(p.x, p.y, p.z, B.c[0], B.c[1], B.c[2], M.ds);
        // Downsample_Storage = Search_by_range(box): live existing points, then the new points accepted so far
        int nE = 0;
        float bd = INFINITY;
        unsigned long long ord = ~0ull;   // visiting order of the best candidate: (brick sequence number << 32 | slot), new points after all bricks
        long long bref = -1;              // >= 0: pool offset of an existing point; <= -2: new point index -(bref+2); -1: none
        unsigned seq = 0;
        for (int kz = B.blo[2]; kz <= B.bhi[2]; kz++)
            for (int ky = B.blo[1]; ky <= B.bhi[1]; ky++)
                for (int kx = B.blo[0]; kx <= B.bhi[0]; kx++, seq++) {
                    unsigned first = 0, count = 0;
                    if (!li_brick_find(M.ent, M.mask, li_pack_key(kx, ky, kz), first, count)) continue;
                    for (unsigned jj = lane; jj < count; jj += 32) {
                        const float4 q = M.pool[(size_t)first + jj];
                        if (__float_as_uint(q.w) == 0xffffffffu || !li_in_box(B, q)) continue;
                        nE++;
                        const float d = li_center_dist_cell(q.x, q.y, q.z, B.c[0], B.c[1], B.c[2], M.ds);
                        if (d < bd) { bd = d; ord = ((unsigned long long)seq << 32) | jj; bref = (long long)first + jj; }
                    }
                }
        for (int e = lane; e < pos; e += 32) {
            const int k = csorted[e];
            if (!ins[k]) continue;
            const float4 q = pts[k];
            if (!li_in_box(B, q)) continue;
            nE++;
            const float d = li_center_dist_cell(q.x, q.y, q.z, B.c[0], B.c[1], B.c[2], M.ds);
            if (d < bd) { bd = d; ord = (1ull << 60) | (unsigned)e; bref = -((long long)k + 2); }
        }
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) {
            nE += __shfl_xor_sync(LI_FULL, nE, o);
            const float d2 = __shfl_xor_sync(LI_FULL, bd, o);
            const unsigned long long o2 = __shfl_xor_sync(LI_FULL, ord, o);
            const long long b2 = __shfl_xor_sync(LI_FULL, bref, o);
            if (d2 < bd || (d2 == bd && o2 < ord)) { bd = d2; ord = o2; bref = b2; }
        }
        float bxx = 0, byy = 0, bzz = 0;
        if (bref >= 0) { const float4 q = M.pool[bref]; bxx = q.x; byy = q.y; bzz = q.z; }
        else if (bref <= -2) { const float4 q = pts[-(bref + 2)]; bxx = q.x; byy = q.y; bzz = q.z; }
        const bool newwins = !(nE > 0 && bd < dp);
        const bool same = newwins || (nE > 0 && fabsf(__fsub_rn(p.x, bxx)) < 1e-6f && fabsf(__fsub_rn(p.y, byy)) < 1e-6f &&
                                      fabsf(__fsub_rn(p.z, bzz)) < 1e-6f);
        if (!(nE > 1 || same)) continue;   // (uniform: every lane holds the same reduced values)
        changed++;
        // Delete_by_range(box), then the winner is (re)inserted
        if (nE > 0) {
            for (int kz = B.blo[2]; kz <= B.bhi[2]; kz++)
                for (int ky = B.blo[1]; ky <= B.bhi[1]; ky++)
                    for (int kx = B.blo[0]; kx <= B.bhi[0]; kx++) {
                        const unsigned long long key = li_pack_key(kx, ky, kz);
                        unsigned first = 0, count = 0;
                        if (!li_brick_find(M.ent, M.mask, key, first, count)) continue;
                        bool any = false;
                        for (unsigned jj = lane; jj < count; jj += 32) {
                            float4* qp = &M.pool[(size_t)first + jj];
                            if (__float_as_uint(qp->w) == 0xffffffffu || !li_in_box(B, *qp)) continue;
                            if (!newwins && bref == (long long)first + jj) continue;
                            qp->w = __uint_as_float(0xffffffffu);
                            any = true;
                        }
                        if (!__any_sync(LI_FULL, any) || lane != 0) continue;
                        unsigned h = li_hash(key) & M.mask;
                        for (unsigned t = 0; t <= M.mask; t++) {
                            unsigned long long k = *reinterpret_cast<volatile unsigned long long*>(&M.ent[h]);
                            if (k == key) { li_touch(M, (int)h); break; }
                            if (k == LI_EMPTY_KEY) break;
                            h = (h + 1) & M.mask;
                        }
                    }
            for (int e = lane; e < pos; e += 32) {
                const int k = csorted[e];
                if (ins[k] && li_in_box(B, pts[k]) && !(!newwins && bref == -((long long)k + 2))) ins[k] = 0;
            }
        }
        if (newwins && lane == 0) ins[cur] = 1;
        __syncwarp();   // the next step reads the tombstones and ins[] this one wrote
    }
    if (changed && lane == 0) atomicAdd(&M.counters[CNT_CHANGED], changed);
}

// pass D3b: append the new points that survived the replay.
__global__ void k_ds_append(MapDev M, const float4* __restrict__ pts, int n, const int* __restrict__ slot_of,
                            const int* __restrict__ ins) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (!ins[i]) return;
    int s = slot_of[i];
    if (s < 0) return;
    uint4 e = M.ent[s];
    if (M.aux[s].y == 0u) return;   // reservation failed (pool full)
    unsigned j = atomicAdd(&M.aux[s].z, 1u);
    float4 p = pts[i];
    int cx = li_cell(p.x, M.ds), cy = li_cell(p.y, M.ds), cz = li_cell(p.z, M.ds);
    unsigned long long key;
    unsigned vib;
    li_storage(M, p, cx, cy, cz, key, vib);
    p.w = __uint_as_float(vib);
    LI_EMUL_ASSERT(e.w + j < M.aux[s].x && (unsigned long long)e.z + M.aux[s].x <= M.pool_cap);
    M.pool[(size_t)e.z + e.w + j] = p;
}

// pass D4: one warp per touched brick -- squeeze out tombstones over [0, count+fill), fix counts.
__global__ void k_ds_compact(MapDev M) {
    const int lane = threadIdx.x & 31;
    const int nw = (gridDim.x * blockDim.x) >> 5, ntouched = M.counters[CNT_TOUCHED];
    for (int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < ntouched; w += nw) {
    int s = M.touched_list[w];
    uint4 e = M.ent[s];
    uint4 a = M.aux[s];
    unsigned total = e.w + a.z;
    unsigned wr = 0;
    for (unsigned base = 0; base < total; base += 32) {
        unsigned j = base + lane;
        float4 q = make_float4(0, 0, 0, 0);
        bool live = false;
        if (j < total) {
            q = M.pool[(size_t)e.z + j];
            live = __float_as_uint(q.w) != 0xffffffffu;
        }
        unsigned mm = __ballot_sync(LI_FULL, live);
        if (live) M.pool[(size_t)e.z + wr + __popc(mm & ((1u << lane) - 1u))] = q;
        wr += __popc(mm);
        __syncwarp();
    }
    if (lane == 0) {
        M.ent[s].w = wr;
        M.aux[s].y = 0u;
        M.aux[s].z = 0u;
        M.aux[s].w = 0u;
        atomicAdd(&M.counters[CNT_LIVE], (int)wr - (int)e.w);
    }
    }
}

// ---- box delete (KD_TREE::Delete_Point_Boxes, ikd_Tree.cpp:500-520 -> Delete_by_range :608-670) -----------------
// A live point is deleted iff some box contains it under the reference's half-open float test
// vertex_min <= c && vertex_max > c on every axis (:633). One warp per hash slot: tombstone-free in-place squeeze.
__global__ void k_map_delete_boxes(MapDev M, unsigned slots, const float* __restrict__ boxes /* n x {min xyz, max xyz} */, int nbox,
                                   int* __restrict__ deleted) {
    int wb = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (wb >= M.counters[CNT_BRICKS]) return;   // `slots` = an upper bound of the brick count (the grid is sized by the host)
    const int w = M.brick_slots[wb];
    uint4 e = M.ent[w];
    unsigned long long k = (unsigned long long)e.x | ((unsigned long long)e.y << 32);
    if (k == LI_EMPTY_KEY || e.w == 0u) return;
    unsigned wr = 0;
    for (unsigned base = 0; base < e.w; base += 32) {
        unsigned j = base + lane;
        float4 q = make_float4(0, 0, 0, 0);
        bool keep = false;
        if (j < e.w) {
            q = M.pool[(size_t)e.z + j];
            keep = true;
            for (int b = 0; b < nbox; b++) {
                const float* bx = boxes + 6 * b;
                if (bx[0] <= q.x && bx[3] > q.x && bx[1] <= q.y && bx[4] > q.y && bx[2] <= q.z && bx[5] > q.z) keep = false;
            }
        }
        unsigned mm = __ballot_sync(LI_FULL, keep);
        if (keep) M.pool[(size_t)e.z + wr + __popc(mm & ((1u << lane) - 1u))] = q;
        wr += __popc(mm);
        __syncwarp();
    }
    if (lane == 0 && wr != e.w) {
        M.ent[w].w = wr;
        atomicAdd(&M.counters[CNT_LIVE], (int)wr - (int)e.w);
        atomicAdd(deleted, (int)(e.w - wr));
    }
}

// The stand-alone 5-NN search (both twins), per query: the ids (pool offsets, -1 = missing) and distances k_knn_queries /
// k_knn_cells_queries left -> the outputs (any may be null), so that results never ship the pool itself. The count is the number of
// ids >= 0. With both xyz and d2 wanted, four passes over the found ranks [0, cnt) swap neighbours whose distances differ by less than
// 1e-10 to smaller x first: the PointType_CMP tie order (ikd_Tree.h:57-60). (Not the plane kernel's tie_order, which bubbles over all
// five ranks with shrinking bounds.)
__global__ void k_query_finish(const float4* __restrict__ pool, const int* __restrict__ ids, const float* __restrict__ d2, int n,
                               float* __restrict__ out_xyz, float* __restrict__ out_d2, int* __restrict__ out_cnt) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float x[5], y[5], z[5], d[5];
    int cnt = 0;
#pragma unroll
    for (int k = 0; k < 5; k++) {
        const int id = ids[(size_t)i * 5 + k];
        const float4 q = (id >= 0) ? pool[id] : make_float4(0.f, 0.f, 0.f, 0.f);
        x[k] = q.x; y[k] = q.y; z[k] = q.z;
        d[k] = d2[(size_t)i * 5 + k];
        if (id >= 0) cnt++;
    }
    if (out_xyz && out_d2) {
#pragma unroll
        for (int pass = 0; pass < 4; pass++) {
#pragma unroll
            for (int k = 0; k < 4; k++) {
                if (k + 1 < cnt && fabsf(d[k] - d[k + 1]) < 1e-10f && x[k + 1] < x[k]) {
                    float t = x[k]; x[k] = x[k + 1]; x[k + 1] = t;
                    t = y[k]; y[k] = y[k + 1]; y[k + 1] = t;
                    t = z[k]; z[k] = z[k + 1]; z[k + 1] = t;
                    t = d[k]; d[k] = d[k + 1]; d[k + 1] = t;
                }
            }
        }
    }
    if (out_cnt) out_cnt[i] = cnt;
#pragma unroll
    for (int k = 0; k < 5; k++) {
        if (out_xyz) {
            float* o = out_xyz + ((size_t)i * 5 + k) * 3;
            o[0] = x[k]; o[1] = y[k]; o[2] = z[k];
        }
        if (out_d2) out_d2[(size_t)i * 5 + k] = d[k];
    }
}

// stores one int in stream order (the point count of a device cloud download)
__global__ void k_store_int(int* __restrict__ p, int v) {
    if (blockIdx.x == 0 && threadIdx.x == 0) *p = v;
}

// ---- flatten -------------------------------------------------------------------------------------
__global__ void k_map_flatten(MapDev M, unsigned slots, float* __restrict__ out, int cap, int* __restrict__ out_n) {
    int wb = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (wb >= M.counters[CNT_BRICKS]) return;   // `slots` = an upper bound of the brick count (the grid is sized by the host)
    const int w = M.brick_slots[wb];
    uint4 e = M.ent[w];
    unsigned long long k = (unsigned long long)e.x | ((unsigned long long)e.y << 32);
    if (k == LI_EMPTY_KEY || e.w == 0u) return;
    int base = 0;
    if (lane == 0) base = atomicAdd(out_n, (int)e.w);
    base = __shfl_sync(LI_FULL, base, 0);
    for (unsigned j = lane; j < e.w; j += 32) {
        int o = base + (int)j;
        if (o < cap) {
            float4 q = M.pool[(size_t)e.z + j];
            out[3 * (size_t)o] = q.x;
            out[3 * (size_t)o + 1] = q.y;
            out[3 * (size_t)o + 2] = q.z;
        }
    }
}

// live points as float4 {x, y, z, 0} (liinit_map_compact re-inserts them into a cleared pool)
__global__ void k_map_flatten4(MapDev M, unsigned slots, float4* __restrict__ out, int cap, int* __restrict__ out_n) {
    int wb = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (wb >= M.counters[CNT_BRICKS]) return;   // `slots` = an upper bound of the brick count (the grid is sized by the host)
    const int w = M.brick_slots[wb];
    uint4 e = M.ent[w];
    unsigned long long k = (unsigned long long)e.x | ((unsigned long long)e.y << 32);
    if (k == LI_EMPTY_KEY || e.w == 0u) return;
    int base = 0;
    if (lane == 0) base = atomicAdd(out_n, (int)e.w);
    base = __shfl_sync(LI_FULL, base, 0);
    for (unsigned j = lane; j < e.w; j += 32) {
        int o = base + (int)j;
        if (o < cap) {
            float4 q = M.pool[(size_t)e.z + j];
            q.w = 0.f;
            out[o] = q;
        }
    }
}

// ---- map_incremental classification (laserMapping.cpp:516-559) ------------------------------------
// flag[i]: 0 = skip, 1 = PointToAdd (downsample insert), 2 = PointNoNeedDownsample (plain insert).
// world[i] = pointBodyToWorld(body[i]) with the FINAL state (:523). near_xyz: Nearest_Points retained from the last search pass
// (copies of the map points, w = 1 / 0 = found / missing rank) -- valid whatever happened to the map since, as in the reference.
__global__ void k_incr_classify(MapDev M, PoseD P, const float4* __restrict__ body, int n, const float4* __restrict__ near_xyz,
                                double ds, int flg_EKF_inited, float4* __restrict__ world, int* __restrict__ flag) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float4 b = body[i];
    float wx, wy, wz;
    li_body_to_world(P, b.x, b.y, b.z, wx, wy, wz);
    world[i] = make_float4(wx, wy, wz, 0.f);
    float4 nb[5];
    int cnt = 0;
#pragma unroll
    for (int j = 0; j < 5; j++) {
        nb[j] = near_xyz[(size_t)i * 5 + j];
        if (nb[j].w != 0.f) cnt++;
    }
    int f = 1;
    if (cnt > 0 && flg_EKF_inited) {
        // mid_point: double expression stored to float (laserMapping.cpp:530-535)
        float mx = (float)__dadd_rn(__dmul_rn(floor(__ddiv_rn((double)wx, ds)), ds), __dmul_rn(0.5, ds));
        float my = (float)__dadd_rn(__dmul_rn(floor(__ddiv_rn((double)wy, ds)), ds), __dmul_rn(0.5, ds));
        float mz = (float)__dadd_rn(__dmul_rn(floor(__ddiv_rn((double)wz, ds)), ds), __dmul_rn(0.5, ds));
        float dist = li_dist2(wx, wy, wz, mx, my, mz);
        float4 n0 = nb[0];
        double half = 0.5 * ds;
        if ((double)fabsf(__fsub_rn(n0.x, mx)) > half && (double)fabsf(__fsub_rn(n0.y, my)) > half &&
            (double)fabsf(__fsub_rn(n0.z, mz)) > half) {
            f = 2;
        } else {
            if (cnt >= 5) {
#pragma unroll
                for (int j = 0; j < 5; j++) {
                    if (li_dist2(nb[j].x, nb[j].y, nb[j].z, mx, my, mz) < dist) f = 0;
                }
            }
        }
    }
    flag[i] = f;
    if (f == 1) atomicAdd(&M.counters[CNT_NADD], 1);
    if (f == 2) atomicAdd(&M.counters[CNT_NNOD], 1);
}
