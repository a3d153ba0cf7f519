// assess_kernels.cuh -- map sharpness of the stored LIO scans under a candidate extrinsic (DESIGN.md section 4d).
//
// Every stored point is placed in the world with li_body_to_world, binned into cubic cells and sorted by cell (the stable radix sort
// of sort_kernels.cuh, extended to 64-bit keys). Every s-th stored point is a query: it sums the fp64 moments of the offsets of every
// stored point within the radius, candidates taken cell by cell in (dz, dy, dx) order and, inside a cell, by ascending stored index.
// The covariance of that neighbourhood gives the point's entropy h = 1/2 ln det(2 pi e Sigma) and plane variance v = lambda_min(Sigma).
// Every query's value is a function of the stored data alone, and the totals are summed in query order by one block, so the results
// are bit-identical from call to call and do not depend on the launch shape or the number of SMs.
// A cloud (liinit_assess_cloud) takes every stored point as a query, in batches of consecutive stored indices over one placement and
// sort, and turns the per-point values into 8-float records, one per point or, summed in stored order, one per occupied cubic leaf.
#pragma once
#include "common.cuh"
#include "sort_kernels.cuh"
#include "preprocess_kernels.cuh"   // li_block_excl_scan, LI_FR_TILE

#define LI_AS_BLOCK 256   // threads of the moments kernel (8 warps)
#define LI_AS_TILE 32     // candidate points a warp stages in shared memory per step
#define LI_AS_COORD_LIMIT 1073741824.0   // |x| / cell edge must stay below 2^30

// The cell grid of one evaluation: bounding box of the occupied cells, cell key = ((z - lo.z) * ext.y + (y - lo.y)) * ext.x + (x - lo.x).
struct AsGrid {
    double edge;        // cell edge: the radius enlarged by 2^-20 (see li_as_cell)
    int lo[3];
    long long ext[3];
};

// Per-query totals of the last evaluation.
struct AsTotals {
    double sum_h, sum_v;
    long long valid, sparse, degenerate;
};

// Cell coordinate of a placed coordinate. The edge is r (1 + 2^-20): a point within r of another lies within one cell of it along every
// axis even after the rounding of the division, so the 27 cells around a query hold all its neighbours.
__device__ __forceinline__ int li_as_cell(float w, double edge, bool& ok) {
    const double q = (double)w / edge;
    ok = fabs(q) < LI_AS_COORD_LIMIT;   // false for NaN and infinities too
    return ok ? (int)floor(q) : 0;
}

__device__ __forceinline__ unsigned long long li_as_key(const AsGrid& G, int x, int y, int z) {
    return ((unsigned long long)(z - G.lo[2]) * (unsigned long long)G.ext[1] + (unsigned long long)(y - G.lo[1])) * (unsigned long long)G.ext[0] +
           (unsigned long long)(x - G.lo[0]);
}

// append: the staged cloud (xyz; w = time) into the store with the scan index in w; thread 0 stores the scan's pose
__global__ void k_as_store(const float4* __restrict__ stage, int n, int scan, PoseD P, float4* __restrict__ dst, PoseD* __restrict__ poses) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) poses[scan] = P;
    if (i >= n) return;
    const float4 p = stage[i];
    dst[i] = make_float4(p.x, p.y, p.z, __int_as_float(scan));
}

// the placement pose of a stored point of scan S: the scan's rot_end / pos_end with the candidate extrinsic (as_run: the scan's own)
__device__ __forceinline__ PoseD li_as_pose(const PoseD& S, int as_run, const PoseD& cand) {
    PoseD P = cand;
#pragma unroll
    for (int k = 0; k < 9; k++) P.R[k] = S.R[k];
#pragma unroll
    for (int k = 0; k < 3; k++) P.p[k] = S.p[k];
    if (as_run) {
#pragma unroll
        for (int k = 0; k < 9; k++) P.RLI[k] = S.RLI[k];
#pragma unroll
        for (int k = 0; k < 3; k++) P.TLI[k] = S.TLI[k];
    }
    return P;
}

// the cells of a placed point: c / C take it as the thread's min / max cell; bad = 1 when it lies outside the cell range
__device__ __forceinline__ void li_as_cells(const float w[3], double edge, int c[3], int C[3], int& bad) {
#pragma unroll
    for (int a = 0; a < 3; a++) {
        bool ok;
        const int v = li_as_cell(w[a], edge, ok);
        bad |= ok ? 0 : 1;
        if (ok) c[a] = C[a] = v;
    }
}

// the warp's min / max cells and bad flag into box[0..2] min cell, [3..5] max cell (atomics, initialised to INT_MAX / INT_MIN by the
// caller), box[6] = 1 when a point lies outside the cell range; every lane of the warp calls it
__device__ __forceinline__ void li_as_box(int c[3], int C[3], int bad, int* __restrict__ box) {
    for (int o = 16; o >= 1; o >>= 1) {
#pragma unroll
        for (int a = 0; a < 3; a++) {
            c[a] = min(c[a], __shfl_xor_sync(LI_FULL, c[a], o));
            C[a] = max(C[a], __shfl_xor_sync(LI_FULL, C[a], o));
        }
        bad |= __shfl_xor_sync(LI_FULL, bad, o);
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int a = 0; a < 3; a++) {
            atomicMin(&box[a], c[a]);
            atomicMax(&box[3 + a], C[a]);
        }
        if (bad) box[6] = 1;
    }
}

// place: every stored point with its scan's pose and the candidate extrinsic (as_run: the scan's own); the cell box as li_as_box
__global__ void k_as_place(const float4* __restrict__ pts, const PoseD* __restrict__ poses, int n, int as_run, PoseD cand, double edge,
                           float4* __restrict__ world, int* __restrict__ box) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    int c[3] = {0x7fffffff, 0x7fffffff, 0x7fffffff}, C[3] = {-0x7fffffff - 1, -0x7fffffff - 1, -0x7fffffff - 1};
    int bad = 0;
    if (i < n) {
        const float4 p = pts[i];
        const PoseD P = li_as_pose(poses[__float_as_int(p.w)], as_run, cand);
        float w[3];
        li_body_to_world(P, p.x, p.y, p.z, w[0], w[1], w[2]);
        world[i] = make_float4(w[0], w[1], w[2], 0.f);
        li_as_cells(w, edge, c, C, bad);
    }
    li_as_box(c, C, bad, box);
}

// keys of the placed points (the cells are computed exactly as in k_as_place) and the identity permutation for the sort
__global__ void k_as_key(const float4* __restrict__ world, int n, AsGrid G, unsigned long long* __restrict__ key, unsigned* __restrict__ klo,
                         unsigned* __restrict__ vals) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 w = world[i];
    bool ok;
    const int x = li_as_cell(w.x, G.edge, ok), y = li_as_cell(w.y, G.edge, ok), z = li_as_cell(w.z, G.edge, ok);
    const unsigned long long k = li_as_key(G, x, y, z);
    key[i] = k;
    klo[i] = (unsigned)k;
    vals[i] = (unsigned)i;
}

// the placed points in sorted order (w = stored index) and their keys
__global__ void k_as_gather(const float4* __restrict__ world, const unsigned long long* __restrict__ key, const unsigned* __restrict__ sv, int n,
                            float4* __restrict__ sorted, unsigned long long* __restrict__ skey) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const unsigned i = sv[p];
    const float4 w = world[i];
    sorted[p] = make_float4(w.x, w.y, w.z, __int_as_float((int)i));
    skey[p] = key[i];
}

// stored point i is a query of the pass: every stride-th point with index in [qa, qb) (an evaluation: [0, n); a cloud: one batch)
__device__ __forceinline__ int li_as_is_query(int i, int stride, int qa, int qb) {
    return i % stride == 0 && i >= qa && i < qb ? 1 : 0;
}

// cell table and query list, step 1 (blockDim.x == LI_FR_TILE): per block the number of cell starts (tc) and of queries (tq); block 0
// zeroes tc[gridDim.x] and tq[gridDim.x], which the exclusive scans turn into the totals
__global__ void k_as_mark(const unsigned long long* __restrict__ skey, const float4* __restrict__ sorted, int n, int stride, int qa, int qb,
                          int* __restrict__ tc, int* __restrict__ tq) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    const int fc = p < n && (p == 0 || skey[p] != skey[p - 1]) ? 1 : 0;
    const int fq = p < n ? li_as_is_query(__float_as_int(sorted[p].w), stride, qa, qb) : 0;
    int t1, t2;
    li_block_excl_scan(fc, &t1);
    __syncthreads();   // li_block_excl_scan's shared words are reused by the second scan
    li_block_excl_scan(fq, &t2);
    if (threadIdx.x == 0) {
        tc[blockIdx.x] = t1;
        tq[blockIdx.x] = t2;
        if (blockIdx.x == 0) tc[gridDim.x] = tq[gridDim.x] = 0;
    }
}

// step 2 (tc, tq: exclusive per-block offsets): cell c starts at sorted position cell_start[c], has key cell_key[c] and its queries are
// qlist[cell_q0[c] .. cell_q0[c + 1]); the sentinels cell_start[ncells] = n and cell_q0[ncells] = queries close the tables
__global__ void k_as_index(const unsigned long long* __restrict__ skey, const float4* __restrict__ sorted, int n, int stride, int qa, int qb,
                           const int* __restrict__ tc, const int* __restrict__ tq, int* __restrict__ cell_start, unsigned long long* __restrict__ cell_key,
                           int* __restrict__ cell_q0, int* __restrict__ qlist) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    const int fc = p < n && (p == 0 || skey[p] != skey[p - 1]) ? 1 : 0;
    const int fq = p < n ? li_as_is_query(__float_as_int(sorted[p].w), stride, qa, qb) : 0;
    int t;
    const int c = tc[blockIdx.x] + li_block_excl_scan(fc, &t);
    __syncthreads();
    const int q = tq[blockIdx.x] + li_block_excl_scan(fq, &t);
    if (fc) {
        cell_start[c] = p;
        cell_key[c] = skey[p];
        cell_q0[c] = q;
    }
    if (fq) qlist[q] = p;
    if (p == 0) {
        cell_start[tc[gridDim.x]] = n;
        cell_q0[tc[gridDim.x]] = tq[gridDim.x];
    }
}

// warp tasks, step 1 (blockDim.x == LI_FR_TILE): a cell with k queries makes ceil(k / 32) tasks of up to 32 queries; per block totals
__global__ void k_as_task_count(const int* __restrict__ cell_q0, const int* __restrict__ ncells, int* __restrict__ tt) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    const int nc = *ncells;
    const int k = c < nc ? (cell_q0[c + 1] - cell_q0[c] + 31) >> 5 : 0;
    int tot;
    li_block_excl_scan(k, &tot);
    if (threadIdx.x == 0) {
        tt[blockIdx.x] = tot;
        if (blockIdx.x == 0) tt[gridDim.x] = 0;
    }
}

// step 2: tasks[j] = {cell, first query (index into qlist), queries}
__global__ void k_as_task_emit(const int* __restrict__ cell_q0, const int* __restrict__ ncells, const int* __restrict__ tt, int4* __restrict__ tasks) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    const int nc = *ncells;
    const int q0 = c < nc ? cell_q0[c] : 0, nq = c < nc ? cell_q0[c + 1] - q0 : 0;
    int tot;
    int j = tt[blockIdx.x] + li_block_excl_scan((nq + 31) >> 5, &tot);
    for (int k = 0; k < nq; k += 32, j++) tasks[j] = make_int4(c, q0 + k, min(32, nq - k), 0);
}

// one Jacobi rotation of the symmetric 3x3 (Numerical Recipes' jacobi): zeroes a_pq; arp / arq are the third row's entries
__device__ __forceinline__ void li_jacobi_rot(double& app, double& aqq, double& apq, double& arp, double& arq, int sweep) {
    if (apq == 0.0) return;
    const double g = 100.0 * fabs(apq);
    if (sweep > 3 && fabs(app) + g == fabs(app) && fabs(aqq) + g == fabs(aqq)) {
        apq = 0.0;
        return;
    }
    const double h = aqq - app;
    double t;
    if (fabs(h) + g == fabs(h)) {
        t = apq / h;
    } else {
        const double theta = 0.5 * h / apq;
        t = 1.0 / (fabs(theta) + sqrt(1.0 + theta * theta));
        if (theta < 0.0) t = -t;
    }
    const double c = 1.0 / sqrt(1.0 + t * t), s = t * c, tau = s / (1.0 + c);
    app -= t * apq;
    aqq += t * apq;
    apq = 0.0;
    const double rp = arp, rq = arq;
    arp = rp - s * (rq + rp * tau);
    arq = rq + s * (rp - rq * tau);
}

// smallest eigenvalue of the symmetric [[a00 a01 a02] [a01 a11 a12] [a02 a12 a22]] by cyclic Jacobi sweeps (small eigenvalues keep their
// relative accuracy, unlike the trigonometric closed form near a double eigenvalue)
__device__ __forceinline__ double li_sym3_min_eig(double a00, double a01, double a02, double a11, double a12, double a22) {
    for (int sweep = 0; sweep < 32; sweep++) {
        if (a01 == 0.0 && a02 == 0.0 && a12 == 0.0) break;
        li_jacobi_rot(a00, a11, a01, a02, a12, sweep);   // (0,1): third row entries a20, a21
        li_jacobi_rot(a00, a22, a02, a01, a12, sweep);   // (0,2): a10, a12
        li_jacobi_rot(a11, a22, a12, a01, a02, sweep);   // (1,2): a01, a02
    }
    return fmin(a00, fmin(a11, a22));
}

#define LI_AS_H0 8.513631199228037   // 3 ln(2 pi e)

// neighbour moments: one warp per task, lanes own the task's queries (all in one cell); the candidate cells are staged through shared
// memory LI_AS_TILE points at a time and every lane runs over every staged point. A dense cell's queries are split over many tasks, and
// the tasks are handed out by a ticket, so no warp carries a dense cell alone. Outputs by query index (stored index / stride): the
// neighbour count, h and v (NaN for a sparse or degenerate neighbourhood).
__global__ void __launch_bounds__(LI_AS_BLOCK) k_as_moments(const float4* __restrict__ sorted, const int* __restrict__ cell_start,
                                                            const unsigned long long* __restrict__ cell_key, const int* __restrict__ ncells_p,
                                                            const int* __restrict__ qlist, const int4* __restrict__ tasks,
                                                            const int* __restrict__ ntasks_p, unsigned* __restrict__ ticket, AsGrid G, double r2,
                                                            int stride, int min_nb, int* __restrict__ qn, double* __restrict__ qh,
                                                            double* __restrict__ qv) {
    __shared__ float4 s_tile[LI_AS_BLOCK / 32][LI_AS_TILE];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int ntasks = *ntasks_p, ncells = *ncells_p;
    for (;;) {
        int t = 0;
        if (lane == 0) t = (int)atomicAdd(ticket, 1u);
        t = __shfl_sync(LI_FULL, t, 0);
        if (t >= ntasks) return;
        const int4 task = tasks[t];
        const bool active = lane < task.z;
        float4 me = make_float4(0.f, 0.f, 0.f, 0.f);
        if (active) me = sorted[qlist[task.y + lane]];
        const double qx = me.x, qy = me.y, qz = me.z;
        const unsigned long long ck = cell_key[task.x];
        const int cx = G.lo[0] + (int)(ck % (unsigned long long)G.ext[0]);
        const int cy = G.lo[1] + (int)((ck / (unsigned long long)G.ext[0]) % (unsigned long long)G.ext[1]);
        const int cz = G.lo[2] + (int)(ck / ((unsigned long long)G.ext[0] * (unsigned long long)G.ext[1]));
        int n = 0;
        double s1x = 0, s1y = 0, s1z = 0, sxx = 0, sxy = 0, sxz = 0, syy = 0, syz = 0, szz = 0;
        for (int d = 0; d < 27; d++) {
            const int x = cx + d % 3 - 1, y = cy + (d / 3) % 3 - 1, z = cz + d / 9 - 1;   // (dz, dy, dx) ascending
            if (x < G.lo[0] || y < G.lo[1] || z < G.lo[2] || x - G.lo[0] >= G.ext[0] || y - G.lo[1] >= G.ext[1] || z - G.lo[2] >= G.ext[2]) continue;
            const unsigned long long k = li_as_key(G, x, y, z);
            int lo = 0, hi = ncells;   // first cell key >= k (every lane searches the same key: broadcast loads)
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (cell_key[mid] < k) lo = mid + 1; else hi = mid;
            }
            if (lo >= ncells || cell_key[lo] != k) continue;
            const int b = cell_start[lo], e = cell_start[lo + 1];
            for (int base = b; base < e; base += LI_AS_TILE) {
                const int m = min(LI_AS_TILE, e - base);
                if (lane < m) s_tile[warp][lane] = sorted[base + lane];
                __syncwarp();
                if (active)
                    for (int j = 0; j < m; j++) {
                        const float4 c = s_tile[warp][j];
                        const double dx = (double)c.x - qx, dy = (double)c.y - qy, dz = (double)c.z - qz;
                        const double d2 = (dx * dx + dy * dy) + dz * dz;
                        if (d2 <= r2) {
                            n++;
                            s1x += dx; s1y += dy; s1z += dz;
                            sxx += dx * dx; sxy += dx * dy; sxz += dx * dz;
                            syy += dy * dy; syz += dy * dz; szz += dz * dz;
                        }
                    }
                __syncwarp();
            }
        }
        if (active) {
            const int qi = __float_as_int(me.w) / stride;
            double h = __longlong_as_double(0x7ff8000000000000ll), v = h;   // NaN: sparse or degenerate
            if (n >= min_nb) {
                const double mx = s1x / n, my = s1y / n, mz = s1z / n;
                const double cxx = sxx / n - mx * mx, cxy = sxy / n - mx * my, cxz = sxz / n - mx * mz;
                const double cyy = syy / n - my * my, cyz = syz / n - my * mz, czz = szz / n - mz * mz;
                const double det = cxx * (cyy * czz - cyz * cyz) - cxy * (cxy * czz - cyz * cxz) + cxz * (cxy * cyz - cyy * cxz);
                if (det > 0.0) {
                    h = 0.5 * (LI_AS_H0 + log(det));
                    v = li_sym3_min_eig(cxx, cxy, cxz, cyy, cyz, czz);
                }
            }
            qn[qi] = n;
            qh[qi] = h;
            qv[qi] = v;
        }
    }
}

// totals in query order (one block of 1024 threads: thread t sums queries t, t + 1024, ..., then a fixed tree), independent of the SMs
__global__ void k_as_reduce(const int* __restrict__ qn, const double* __restrict__ qh, const double* __restrict__ qv, int nq, int min_nb,
                            AsTotals* __restrict__ out) {
    __shared__ double s_h[1024], s_v[1024];
    __shared__ long long s_c[3][1024];
    const int t = threadIdx.x;
    double h = 0.0, v = 0.0;
    long long nv = 0, ns = 0, nd = 0;
    for (int q = t; q < nq; q += blockDim.x) {
        if (qn[q] < min_nb) {
            ns++;
        } else if (qh[q] != qh[q]) {
            nd++;
        } else {
            nv++;
            h += qh[q];
            v += qv[q];
        }
    }
    s_h[t] = h; s_v[t] = v; s_c[0][t] = nv; s_c[1][t] = ns; s_c[2][t] = nd;
    __syncthreads();
    for (int o = blockDim.x >> 1; o > 0; o >>= 1) {
        if (t < o) {
            s_h[t] += s_h[t + o]; s_v[t] += s_v[t + o];
            s_c[0][t] += s_c[0][t + o]; s_c[1][t] += s_c[1][t + o]; s_c[2][t] += s_c[2][t + o];
        }
        __syncthreads();
    }
    if (t == 0) {
        out->sum_h = s_h[0];
        out->sum_v = s_v[0];
        out->valid = s_c[0][0];
        out->sparse = s_c[1][0];
        out->degenerate = s_c[2][0];
    }
}

// ---- the per-point cloud (liinit_assess_cloud, DESIGN.md section 4d) ----
// Every stored point is a query: the moments above run in batches of consecutive stored indices and write the per-point n, h, v by stored
// index. A record is 8 floats: x y z entropy plane_variance neighbors points valid.

// one record per stored point a + j, j < m, from the placed point and its per-point values (valid: h is not NaN)
__global__ void k_ac_point_rec(const float4* __restrict__ world, const double* __restrict__ qh, const double* __restrict__ qv,
                               const int* __restrict__ qn, int a, int m, float4* __restrict__ rec) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const int i = a + j;
    const float4 w = world[i];
    const double h = qh[i];
    rec[2 * j] = make_float4(w.x, w.y, w.z, (float)h);
    rec[2 * j + 1] = make_float4((float)qv[i], (float)qn[i], 1.f, h == h ? 1.f : 0.f);
}

// the per-point values as they go into a record (h, v, neighbours, valid), for the leaf sums
__global__ void k_ac_point_pack(const double* __restrict__ qh, const double* __restrict__ qv, const int* __restrict__ qn, int n,
                                float4* __restrict__ hvn) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double h = qh[i];
    hvn[i] = make_float4((float)h, (float)qv[i], (float)qn[i], h == h ? 1.f : 0.f);
}

// leaf table, step 1 (blockDim.x == LI_FR_TILE): per block the number of leaf starts in the sorted order perm; block 0 zeroes tl[gridDim.x]
__global__ void k_ac_leaf_mark(const unsigned long long* __restrict__ key, const unsigned* __restrict__ perm, int n, int* __restrict__ tl) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    const int f = p < n && (p == 0 || key[perm[p]] != key[perm[p - 1]]) ? 1 : 0;
    int t;
    li_block_excl_scan(f, &t);
    if (threadIdx.x == 0) {
        tl[blockIdx.x] = t;
        if (blockIdx.x == 0) tl[gridDim.x] = 0;
    }
}

// step 2 (tl: exclusive per-block offsets): leaf c covers sorted positions leaf_start[c] .. leaf_start[c + 1]; the sentinel
// leaf_start[leaves] = n closes the table
__global__ void k_ac_leaf_index(const unsigned long long* __restrict__ key, const unsigned* __restrict__ perm, int n, const int* __restrict__ tl,
                                int* __restrict__ leaf_start) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    const int f = p < n && (p == 0 || key[perm[p]] != key[perm[p - 1]]) ? 1 : 0;
    int t;
    const int c = tl[blockIdx.x] + li_block_excl_scan(f, &t);
    if (f) leaf_start[c] = p;
    if (p == 0) leaf_start[tl[gridDim.x]] = n;
}

// one record per leaf c0 + j, j < m: one thread sums the leaf's points in stored order (the sort is stable over the identity permutation)
// in fp64; centroid and mean neighbour count over all of them, mean h and v over the valid ones (NaN when there is none)
__global__ void k_ac_leaf_rec(const float4* __restrict__ world, const float4* __restrict__ hvn, const unsigned* __restrict__ perm,
                              const int* __restrict__ leaf_start, int c0, int m, float4* __restrict__ rec) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const int b = leaf_start[c0 + j], e = leaf_start[c0 + j + 1];
    double sx = 0.0, sy = 0.0, sz = 0.0, sh = 0.0, sv = 0.0, sn = 0.0;
    int nv = 0;
    for (int p = b; p < e; p++) {
        const unsigned i = perm[p];
        const float4 w = world[i], a = hvn[i];
        sx += w.x; sy += w.y; sz += w.z;
        sn += a.z;
        if (a.w != 0.f) {
            sh += a.x; sv += a.y;
            nv++;
        }
    }
    const double np = (double)(e - b);
    const float nan = __int_as_float(0x7fc00000);
    rec[2 * j] = make_float4((float)(sx / np), (float)(sy / np), (float)(sz / np), nv ? (float)(sh / nv) : nan);
    rec[2 * j + 1] = make_float4(nv ? (float)(sv / nv) : nan, (float)(sn / np), (float)(e - b), (float)nv);
}
