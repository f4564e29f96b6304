// kba_lidar.cu -- lidar depth extraction on sm_90a (BASELINE config 4; C ABI: kba_lidar_depth_batch and kba_lidar_depth, its
// one-view case, in kba_b200.h; the frame step's lidar form, kba_track_frame_step_lidar, runs the same plan and kernels from
// kba_api.cu through kba_kernels.h).  A call works on "views": a cloud seen by one camera with one feature list.  Per-view
// parameters live in a device array; each view's cell counts, starts and cursors sit at its own offset of one concatenated
// array, and its sorted point records in a segment of its cloud's n_points.
//   k_lidar_bin<false>: all (view, point) pairs: project the cloud (coalesced float loads), count points per 16x16-pixel cell
//   k_lidar_scan      : one CTA per view: exclusive scan of its cell counts
//   k_lidar_bin<true> : project again and scatter (u, v, x, y, z, index) into each view's cell-sorted order
//   k_lidar_feature   : one warp per feature of all views: gather the pixel rectangle from the overlapping cells, depth
//                       histogram, largest triangle, plane / view-ray intersection, depth gates; templated on where a feature
//                       reads (u, v) and writes its depth (the batch's packed features, or the frame step's staged rows)
// The bin passes map a block to its view by a per-view block-offset prefix (binary search), the feature pass a warp by the
// feature-offset prefix: no CTA idles on a view smaller than the largest.
// Compiled with -fmad=false: the arithmetic is single precision with the operation order of the specification so that the
// discrete decisions (rectangle membership, histogram bin, arg-max triangle) do not depend on FMA contraction.
#include <algorithm>
#include <climits>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include <cuda_runtime.h>

#include "kba_b200.h"
#include "kba_kernels.h"

namespace {

using kba::LidarParams;

constexpr int kCell = 16;      // pixels per cell side
constexpr int kMaxNb = 96;     // neighbours kept per feature
constexpr int kBins = 64;

struct ProjPt { float u, v, x, y, z; int idx; };

// the segment of x in a prefix off[0] = 0 <= ... <= off[n] with x < off[n]: the largest s < n with off[s] <= x (empty
// segments are skipped)
__device__ __forceinline__ int segment_of(const int* __restrict__ off, int n, int x) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (off[mid] <= x) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__device__ __forceinline__ bool project(const LidarParams& P, const float* __restrict__ p, ProjPt& o) {
    const float x = P.R[0] * p[0] + P.R[1] * p[1] + P.R[2] * p[2] + P.t[0];
    const float y = P.R[3] * p[0] + P.R[4] * p[1] + P.R[5] * p[2] + P.t[1];
    const float z = P.R[6] * p[0] + P.R[7] * p[1] + P.R[8] * p[2] + P.t[2];
    if (!(z > 0.0f)) return false;
    const float u = P.f * x / z + P.cx, v = P.f * y / z + P.cy;
    if (!(u >= 0.0f && u < (float)P.width && v >= 0.0f && v < (float)P.height)) return false;
    o.u = u; o.v = v; o.x = x; o.y = y; o.z = z;
    return true;
}

// blk_off[n_views + 1]: blocks of 256 points per view
template <bool kFill>
__global__ void __launch_bounds__(256) k_lidar_bin(const LidarParams* __restrict__ par, const int* __restrict__ blk_off, int n_views,
                                                   const float* __restrict__ clouds, int* __restrict__ cell_count,
                                                   const int* __restrict__ cell_start, int* __restrict__ cell_cursor,
                                                   ProjPt* __restrict__ sorted) {
    const int view = segment_of(blk_off, n_views, blockIdx.x);
    const LidarParams& P = par[view];
    const int i = (blockIdx.x - blk_off[view]) * blockDim.x + threadIdx.x;
    if (i >= P.n_points) return;
    ProjPt q;
    if (!project(P, clouds + P.cloud_off + (size_t)i * P.stride, q)) return;
    const int cell = P.cell_off + ((int)q.v / kCell) * P.cells_x + ((int)q.u / kCell);
    if (!kFill) {
        atomicAdd(&cell_count[cell], 1);
    } else {
        q.idx = i;
        sorted[P.sort_off + cell_start[cell] + atomicAdd(&cell_cursor[cell], 1)] = q;
    }
}

// one CTA per view; a view's starts are relative to its sorted segment
__global__ void __launch_bounds__(1024) k_lidar_scan(const LidarParams* __restrict__ par, const int* __restrict__ cell_count,
                                                     int* __restrict__ cell_start) {
    __shared__ int s_part[1024];
    const LidarParams& P = par[blockIdx.x];
    const int* cnt = cell_count + P.cell_off;
    int* start = cell_start + P.cell_off;
    const int ncell = P.cells_x * P.cells_y;
    const int per = (ncell + 1023) / 1024, b0 = threadIdx.x * per;
    int s = 0;
    for (int c = b0; c < min(ncell, b0 + per); ++c) s += cnt[c];
    s_part[threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        int acc = 0;
        for (int q = 0; q < 1024; ++q) { const int v = s_part[q]; s_part[q] = acc; acc += v; }
    }
    __syncthreads();
    int acc = s_part[threadIdx.x];
    for (int c = b0; c < min(ncell, b0 + per); ++c) { start[c] = acc; acc += cnt[c]; }
    if (threadIdx.x == 1023) start[ncell] = acc;
}

__device__ __forceinline__ int bin_of(float z, float zmin, float bw) {
    int b = (int)floorf((z - zmin) / bw);
    return b > kBins - 1 ? kBins - 1 : b;
}

// the feature pass's addressing: where feature k reads its (u, v) and writes its depth
struct PackedFeatures {        // kba_lidar_depth_batch: (u, v) pairs and depths in feature order
    const float* __restrict__ uv;
    float* __restrict__ out;
    __device__ __forceinline__ void load(int k, float& fu, float& fv) const { fu = uv[2 * (size_t)k]; fv = uv[2 * (size_t)k + 1]; }
    __device__ __forceinline__ void store(int k, float d) const { out[k] = d; }
};
struct StagedFeatures {        // the frame step: feature k is staged measurement idx[k] (kba::LidarStaged)
    kba::LidarStaged s;
    __device__ __forceinline__ void load(int k, float& fu, float& fv) const {
        const int m = __ldg(s.idx + k);
        fu = __ldg(s.u + m); fv = __ldg(s.v + m);
    }
    __device__ __forceinline__ void store(int k, float d) const {
        s.d[__ldg(s.idx + k)] = d;
        if (k < s.n_copy) s.copy[k] = d;
    }
};

// feat_off[n_views + 1]: the views' features concatenated, n_feats in all.  The result does not depend on the order in which
// the fill pass's atomics placed the points inside a cell: the histogram counts and the nearest depth are order-free, the
// largest triangle is chosen by area and then by the points' original indices, and a rectangle with more than kMaxNb points
// gives -1 whatever was gathered.  That is what makes the depths bit-identical to the sequential specification, whichever
// addressing the features come with.
template <class Feats>
__global__ void __launch_bounds__(128) k_lidar_feature(const LidarParams* __restrict__ par, const int* __restrict__ feat_off,
                                                       int n_views, const ProjPt* __restrict__ sorted_all,
                                                       const int* __restrict__ cell_start_all, const Feats feats, int n_feats) {
    __shared__ ProjPt s_nb[4][kMaxNb];
    __shared__ int s_cnt[4][kBins];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int k = blockIdx.x * 4 + warp;
    if (k >= n_feats) return;
    const LidarParams P = par[segment_of(feat_off, n_views, k)];  // a copy: read through a reference it spills (ptxas -v)
    const ProjPt* sorted = sorted_all + P.sort_off;
    const int* cell_start = cell_start_all + P.cell_off;
    ProjPt* nb = s_nb[warp];
    int* cnt = s_cnt[warp];
    float fu, fv;
    feats.load(k, fu, fv);
    const float cu = fu + P.offx, cv = fv + P.offy;
    // ---- gather the rectangle ----
    const int cx0 = max(0, (int)floorf((cu - P.hw) / kCell)), cx1 = min(P.cells_x - 1, (int)floorf((cu + P.hw) / kCell));
    const int cy0 = max(0, (int)floorf((cv - P.hh) / kCell)), cy1 = min(P.cells_y - 1, (int)floorf((cv + P.hh) / kCell));
    int m = 0;
    for (int cy = cy0; cy <= cy1; ++cy)
        for (int cxi = cx0; cxi <= cx1; ++cxi) {
            const int c = cy * P.cells_x + cxi;
            const int e0 = cell_start[c], e1 = cell_start[c + 1];
            for (int e = e0; e < e1; e += 32) {
                ProjPt q;
                bool in = false;
                if (e + lane < e1) {
                    q = sorted[e + lane];
                    in = fabsf(q.u - cu) <= P.hw && fabsf(q.v - cv) <= P.hh;
                }
                const unsigned mask = __ballot_sync(0xffffffffu, in);
                const int pos = m + __popc(mask & ((1u << lane) - 1));
                if (in && pos < kMaxNb) nb[pos] = q;
                m += __popc(mask);
            }
        }
    __syncwarp();
    float result = -1.0f;
    if (m >= P.min_points && m <= kMaxNb) {
        // ---- depth histogram from the nearest point ----
        float zmin = 3.0e38f;
        for (int i = lane; i < m; i += 32) zmin = fminf(zmin, nb[i].z);
        for (int o = 16; o > 0; o >>= 1) zmin = fminf(zmin, __shfl_xor_sync(0xffffffffu, zmin, o));
        for (int b = lane; b < kBins; b += 32) cnt[b] = 0;
        __syncwarp();
        for (int i = lane; i < m; i += 32) atomicAdd(&cnt[bin_of(nb[i].z, zmin, P.bw)], 1);
        __syncwarp();
        int sel = -1;
        for (int b = 0; b < kBins; ++b) {
            const int c = cnt[b];
            if (c < P.hist_min_count || c == 0) continue;
            const int left = b > 0 ? cnt[b - 1] : -1, right = b < kBins - 1 ? cnt[b + 1] : -1;
            if (c > left && c >= right) { sel = b; break; }
        }
        if (sel >= 0 && cnt[sel] >= P.min_points) {
            // ---- largest triangle (i < j < k by original index), lanes stride over ordered pairs ----
            float best_area = -1.0f;
            int b0 = 0x7fffffff, b1 = 0x7fffffff, b2 = 0x7fffffff, l0 = -1, l1 = -1, l2 = -1;
            for (int pr = lane; pr < m * m; pr += 32) {
                const int i = pr / m, j = pr - i * m;
                if (nb[j].idx <= nb[i].idx) continue;
                if (bin_of(nb[i].z, zmin, P.bw) != sel || bin_of(nb[j].z, zmin, P.bw) != sel) continue;
                const float ax = nb[j].x - nb[i].x, ay = nb[j].y - nb[i].y, az = nb[j].z - nb[i].z;
                for (int q = 0; q < m; ++q) {
                    if (nb[q].idx <= nb[j].idx || bin_of(nb[q].z, zmin, P.bw) != sel) continue;
                    const float bx = nb[q].x - nb[i].x, by = nb[q].y - nb[i].y, bz = nb[q].z - nb[i].z;
                    const float cx = ay * bz - az * by, cy = az * bx - ax * bz, cz = ax * by - ay * bx;
                    const float area = cx * cx + cy * cy + cz * cz;
                    const int a0 = nb[i].idx, a1 = nb[j].idx, a2 = nb[q].idx;
                    bool better = area > best_area;
                    if (!better && area == best_area) better = (a0 < b0) || (a0 == b0 && (a1 < b1 || (a1 == b1 && a2 < b2)));
                    if (better) { best_area = area; b0 = a0; b1 = a1; b2 = a2; l0 = i; l1 = j; l2 = q; }
                }
            }
            for (int o = 16; o > 0; o >>= 1) {
                const float oa = __shfl_xor_sync(0xffffffffu, best_area, o);
                const int o0 = __shfl_xor_sync(0xffffffffu, b0, o), o1 = __shfl_xor_sync(0xffffffffu, b1, o), o2 = __shfl_xor_sync(0xffffffffu, b2, o);
                const int p0 = __shfl_xor_sync(0xffffffffu, l0, o), p1 = __shfl_xor_sync(0xffffffffu, l1, o), p2 = __shfl_xor_sync(0xffffffffu, l2, o);
                bool better = oa > best_area;
                if (!better && oa == best_area) better = (o0 < b0) || (o0 == b0 && (o1 < b1 || (o1 == b1 && o2 < b2)));
                if (better) { best_area = oa; b0 = o0; b1 = o1; b2 = o2; l0 = p0; l1 = p1; l2 = p2; }
            }
            if (lane == 0 && l0 >= 0) {
                const ProjPt A = nb[l0], B = nb[l1], Cc = nb[l2];
                const float e[3][3] = {{B.x - A.x, B.y - A.y, B.z - A.z}, {Cc.x - B.x, Cc.y - B.y, Cc.z - B.z}, {A.x - Cc.x, A.y - Cc.y, A.z - Cc.z}};
                float len[3];
                for (int q = 0; q < 3; ++q) len[q] = sqrtf(e[q][0] * e[q][0] + e[q][1] * e[q][1] + e[q][2] * e[q][2]);
                bool ok = true;
                for (int q = 0; q < 3 && ok; ++q) {
                    const int r = (q + 1) % 3;
                    if (!(len[q] > 0.0f) || !(len[r] > 0.0f)) { ok = false; break; }
                    const float cx = e[q][1] * e[r][2] - e[q][2] * e[r][1], cy = e[q][2] * e[r][0] - e[q][0] * e[r][2], cz = e[q][0] * e[r][1] - e[q][1] * e[r][0];
                    if (sqrtf(cx * cx + cy * cy + cz * cz) / (len[q] * len[r]) < P.crossnorm_min) ok = false;
                }
                if (ok) {
                    float nx = e[0][1] * (-e[2][2]) - e[0][2] * (-e[2][1]), ny = e[0][2] * (-e[2][0]) - e[0][0] * (-e[2][2]), nz = e[0][0] * (-e[2][1]) - e[0][1] * (-e[2][0]);
                    const float nn = sqrtf(nx * nx + ny * ny + nz * nz);
                    nx /= nn; ny /= nn; nz /= nn;
                    const float rx = (fu - P.cx) / P.f, ry = (fv - P.cy) / P.f, rz = 1.0f;
                    const float rl = sqrtf(rx * rx + ry * ry + rz * rz);
                    const float ndr = nx * rx + ny * ry + nz * rz;
                    if (!(fabsf(ndr) / rl < P.viewray_min)) {
                        const float depth = (nx * A.x + ny * A.y + nz * A.z) / ndr;
                        bool good = (depth >= P.depth_min) && (depth <= P.depth_max);
                        if (good && P.local_enabled) {
                            float smin = 0.f, smax = 0.f;
                            bool first = true;
                            for (int i = 0; i < m; ++i) {
                                if (bin_of(nb[i].z, zmin, P.bw) != sel) continue;
                                if (first) { smin = smax = nb[i].z; first = false; }
                                smin = fminf(smin, nb[i].z); smax = fmaxf(smax, nb[i].z);
                            }
                            if (depth < smin * (1.0f - P.local_tol) || depth > smax * (1.0f + P.local_tol)) good = false;
                        }
                        if (good) result = depth;
                    }
                }
            }
        }
    }
    if (lane == 0) feats.store(k, result);
}

void quat_R(const double* q, float* R) {
    const double w = q[0], x = q[1], y = q[2], z = q[3];
    const double M[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y), 2 * (x * y + w * z), 1 - 2 * (x * x + z * z),
                         2 * (y * z - w * x), 2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)};
    for (int i = 0; i < 9; ++i) R[i] = (float)M[i];
}

// a view's pose, intrinsics and options in the kernels' single precision; a negative image size has no cells
void view_params(const double* T, const double* intr, const kba_lidar_options* o, LidarParams& P) {
    quat_R(T, P.R);
    P.t[0] = (float)T[4]; P.t[1] = (float)T[5]; P.t[2] = (float)T[6];
    P.f = (float)intr[0]; P.cx = (float)intr[1]; P.cy = (float)intr[2];
    P.width = o->image_width; P.height = o->image_height;
    P.cells_x = std::max(0, (P.width + kCell - 1) / kCell); P.cells_y = std::max(0, (P.height + kCell - 1) / kCell);
    P.hw = 0.5f * (float)o->rect_width; P.hh = 0.5f * (float)o->rect_height;
    P.offx = (float)o->rect_offset_x; P.offy = (float)o->rect_offset_y; P.bw = (float)o->hist_bin_width;
    P.hist_min_count = o->hist_min_count; P.min_points = o->min_points;
    P.depth_min = (float)o->depth_min; P.depth_max = (float)o->depth_max;
    P.local_enabled = o->local_rel_tolerance >= 0; P.local_tol = (float)o->local_rel_tolerance;
    P.crossnorm_min = (float)o->triangle_crossnorm_min; P.viewray_min = (float)o->viewray_plane_min;
}

size_t al(size_t b) { return (b + 255) & ~(size_t)255; }

// the workspace's scratch: cell counts, cursors and starts (each of cell_bytes), sorted point records
size_t cell_bytes(const kba::LidarPlan& p) { return al(sizeof(int) * (size_t)p.cells); }
size_t sorted_bytes(const kba::LidarPlan& p) { return al(sizeof(ProjPt) * (size_t)std::max(p.pairs, 1LL)); }

// the launch sequence of plan p, its pack() at d_pack, on a workspace whose clouds are copied ahead of it on s
template <class Feats>
cudaError_t launch_lidar(const kba::LidarPlan& p, const kba::LidarWs& ws, const void* d_pack, const Feats& f, cudaStream_t s) {
    const int nw = (int)p.par.size();
    const LidarParams* d_par = (const LidarParams*)d_pack;
    const int* d_blk = (const int*)(d_par + nw);
    const int* d_fo = d_blk + nw + 1;
    ProjPt* sorted = (ProjPt*)ws.sorted;
    const cudaError_t e = cudaMemsetAsync(ws.cnt, 0, 2 * cell_bytes(p), s);  // the cursors follow the counts
    if (e != cudaSuccess) return e;
    if (p.blocks > 0) k_lidar_bin<false><<<(unsigned)p.blocks, 256, 0, s>>>(d_par, d_blk, nw, ws.clouds, ws.cnt, nullptr, nullptr, nullptr);
    k_lidar_scan<<<nw, 1024, 0, s>>>(d_par, ws.cnt, ws.start);
    if (p.blocks > 0) k_lidar_bin<true><<<(unsigned)p.blocks, 256, 0, s>>>(d_par, d_blk, nw, ws.clouds, ws.cnt, ws.start, ws.cur, sorted);
    k_lidar_feature<Feats><<<(unsigned)((p.feats + 3) / 4), 128, 0, s>>>(d_par, d_fo, nw, sorted, ws.start, f, (int)p.feats);
    return cudaSuccess;
}

}  // namespace

extern "C" void kba_lidar_default_options(kba_lidar_options* o) {
    if (!o) return;
    *o = kba_lidar_options{};
    o->image_width = 1242; o->image_height = 375;
    o->rect_width = 6; o->rect_height = 9; o->rect_offset_x = 0; o->rect_offset_y = 0;
    o->hist_bin_width = 0.3; o->hist_min_count = 1; o->min_points = 3;
    o->depth_min = 0; o->depth_max = 100; o->local_rel_tolerance = 0.5;
    o->triangle_crossnorm_min = 0.1; o->viewray_plane_min = 0.1;
}

// implemented in kba_api.cu
extern "C" int kba_internal_stream(kba_handle* h, cudaStream_t* s, int* device);
extern "C" int kba_internal_fail(int code, const char* msg);
extern "C" int kba_internal_workspace(kba_handle* h, size_t bytes, void** out);

namespace kba {

int LidarPlan::add(int c, const kba_lidar_cloud& cl, const double* T, const double* intr, const kba_lidar_options* o, int n_feat) {
    if (cloud_off[c] < 0) {
        cloud_off[c] = (long long)(b_clouds / sizeof(float));
        b_clouds += al(sizeof(float) * (size_t)cl.n_points * cl.stride);
    }
    LidarParams P;
    view_params(T, intr, o, P);
    P.cloud_off = cloud_off[c]; P.n_points = cl.n_points; P.stride = cl.stride;
    P.cell_off = (int)std::min<long long>(cells, INT_MAX); P.sort_off = (int)std::min<long long>(pairs, INT_MAX);
    cells += (long long)P.cells_x * P.cells_y + 1;
    pairs += cl.n_points;
    blocks += (cl.n_points + 255) / 256;
    feats += n_feat;
    if (cells > INT_MAX || pairs > INT_MAX || 2 * feats > INT_MAX) return KBA_ERR_CAPACITY;
    par.push_back(P);
    blk_off.push_back((int)blocks); feat_off.push_back((int)feats);
    return KBA_OK;
}

size_t LidarPlan::pack_bytes() const { return sizeof(LidarParams) * par.size() + 2 * sizeof(int) * (par.size() + 1); }

void LidarPlan::pack(void* dst) const {
    char* d = (char*)dst;
    const size_t nw = par.size();
    memcpy(d, par.data(), sizeof(LidarParams) * nw); d += sizeof(LidarParams) * nw;
    memcpy(d, blk_off.data(), sizeof(int) * (nw + 1)); d += sizeof(int) * (nw + 1);
    memcpy(d, feat_off.data(), sizeof(int) * (nw + 1));
}

// one device workspace owned by the handle (grow-only): clouds | cell counts | cursors | starts | sorted point records | extra
int lidar_workspace(kba_handle* h, const LidarPlan& p, size_t extra, LidarWs& ws) {
    const size_t b_cell = cell_bytes(p), b_sorted = sorted_bytes(p);
    void* base = nullptr;
    if (kba_internal_workspace(h, p.b_clouds + 3 * b_cell + b_sorted + al(extra), &base) != KBA_OK) return KBA_ERR_CUDA;
    char* wp = (char*)base;
    ws.clouds = (float*)wp; wp += p.b_clouds;
    ws.cnt = (int*)wp; wp += b_cell;
    ws.cur = (int*)wp; wp += b_cell;
    ws.start = (int*)wp; wp += b_cell;
    ws.sorted = wp; wp += b_sorted;
    ws.extra = wp;
    return KBA_OK;
}

cudaError_t lidar_copy_clouds(const LidarPlan& p, const kba_lidar_cloud* clouds, const LidarWs& ws, cudaStream_t s) {
    for (size_t c = 0; c < p.cloud_off.size(); ++c) {
        if (p.cloud_off[c] < 0 || clouds[c].n_points == 0) continue;
        const cudaError_t e = cudaMemcpyAsync(ws.clouds + p.cloud_off[c], clouds[c].points,
                                              sizeof(float) * (size_t)clouds[c].n_points * clouds[c].stride, cudaMemcpyHostToDevice, s);
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

cudaError_t launch_lidar_staged(const LidarPlan& p, const LidarWs& ws, const void* d_pack, const LidarStaged& f, cudaStream_t s) {
    return launch_lidar(p, ws, d_pack, StagedFeatures{f}, s);
}

}  // namespace kba

namespace {

int fail_at(int code, const char* fn, const char* what, long long i, const char* msg) {
    const std::string m = std::string(fn) + ": " + what + " " + std::to_string(i) + ": " + msg;
    return kba_internal_fail(code, m.c_str());
}

// the host code of every lidar depth batch: opts[0] for every view, or opts[i] for view i (per_view)
int lidar_batch(kba_handle* h, int32_t n_clouds, const kba_lidar_cloud* clouds, int32_t n_views, const kba_lidar_view* views,
                const kba_lidar_options* opts, bool per_view, float* device_ms, const char* fn) {
    const std::string name(fn);
    if (!h) return kba_internal_fail(KBA_ERR_BAD_ARG, (name + ": null handle").c_str());
    if (n_clouds < 0 || n_views < 0) return kba_internal_fail(KBA_ERR_BAD_ARG, (name + ": negative cloud or view count").c_str());
    if ((n_clouds > 0 && !clouds) || (n_views > 0 && !views)) return kba_internal_fail(KBA_ERR_BAD_ARG, (name + ": null clouds or views").c_str());
    // ---- validation: views, then the clouds the working views name, then the 32-bit totals ----
    std::vector<int> work;
    for (int i = 0; i < n_views; ++i) {
        const kba_lidar_view& v = views[i];
        if (v.n_features < 0) return fail_at(KBA_ERR_BAD_ARG, fn, "view", i, "negative n_features");
        if (v.n_features == 0) continue;
        if (v.cloud < 0 || v.cloud >= n_clouds) return fail_at(KBA_ERR_BAD_ARG, fn, "view", i, "cloud index out of range");
        if (!v.T_cam_lidar || !v.intr || !v.features_uv || !v.depth_out) return fail_at(KBA_ERR_BAD_ARG, fn, "view", i, "null pointer");
        work.push_back(i);
    }
    if (work.empty()) {
        if (device_ms) *device_ms = 0.0f;
        return KBA_OK;
    }
    if (!opts) return kba_internal_fail(KBA_ERR_BAD_ARG, (name + ": null options").c_str());
    std::vector<char> named(n_clouds, 0);
    for (int i : work) {
        const int c = views[i].cloud;
        if (named[c]) continue;
        named[c] = 1;
        const kba_lidar_cloud& cl = clouds[c];
        if (cl.n_points < 0) return fail_at(KBA_ERR_BAD_ARG, fn, "cloud", c, "negative n_points");
        if (cl.stride < 3) return fail_at(KBA_ERR_BAD_ARG, fn, "cloud", c, "stride < 3");
        if (cl.n_points > 0 && !cl.points) return fail_at(KBA_ERR_BAD_ARG, fn, "cloud", c, "null points");
    }
    kba::LidarPlan plan(n_clouds);
    for (int i : work) {
        const kba_lidar_view& v = views[i];
        if (plan.add(v.cloud, clouds[v.cloud], v.T_cam_lidar, v.intr, per_view ? &opts[i] : opts, v.n_features) != KBA_OK)
            return fail_at(KBA_ERR_CAPACITY, fn, "view", i, "the call's cells, (view, point) pairs or features exceed 32-bit indexing");
    }
    const int nw = (int)work.size();
    const size_t feats = (size_t)plan.feats;
    cudaStream_t s;
    int device;
    if (kba_internal_stream(h, &s, &device) != KBA_OK) return KBA_ERR_BAD_ARG;
    // the workspace's extra part: the packed upload (view parameters and prefixes | features) | depths
    const size_t b_par = al(plan.pack_bytes()), b_pack = b_par + al(sizeof(float) * 2 * feats);
    kba::LidarWs ws;
    if (kba::lidar_workspace(h, plan, b_pack + al(sizeof(float) * feats), ws) != KBA_OK) return KBA_ERR_CUDA;
    char* d_pack = (char*)ws.extra;
    float* d_out = (float*)(d_pack + b_pack);
    // host staging of the packed upload and of the depths, grow-only per host thread
    static thread_local std::vector<char> pack;
    static thread_local std::vector<float> depths;
    if (pack.size() < b_pack) pack.resize(b_pack);
    if (depths.size() < feats) depths.resize(feats);
    plan.pack(pack.data());
    for (int w = 0; w < nw; ++w) {
        const kba_lidar_view& v = views[work[w]];
        memcpy(pack.data() + b_par + sizeof(float) * 2 * (size_t)plan.feat_off[w], v.features_uv, sizeof(float) * 2 * (size_t)v.n_features);
    }
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    cudaError_t err = cudaSuccess;
    auto chk = [&](cudaError_t e) { if (err == cudaSuccess && e != cudaSuccess) err = e; };
    chk(cudaSetDevice(device));
    if (device_ms) { chk(cudaEventCreate(&e0)); chk(cudaEventCreate(&e1)); }
    if (err == cudaSuccess) {
        chk(kba::lidar_copy_clouds(plan, clouds, ws, s));
        chk(cudaMemcpyAsync(d_pack, pack.data(), b_pack, cudaMemcpyHostToDevice, s));
        if (e0) chk(cudaEventRecord(e0, s));
        if (err == cudaSuccess) chk(launch_lidar(plan, ws, d_pack, PackedFeatures{(const float*)(d_pack + b_par), d_out}, s));
        if (e1) chk(cudaEventRecord(e1, s));
        chk(cudaMemcpyAsync(depths.data(), d_out, sizeof(float) * feats, cudaMemcpyDeviceToHost, s));
        chk(cudaStreamSynchronize(s));
        chk(cudaGetLastError());
        if (err == cudaSuccess && device_ms) chk(cudaEventElapsedTime(device_ms, e0, e1));
    }
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
    if (err != cudaSuccess) return kba_internal_fail(KBA_ERR_CUDA, cudaGetErrorString(err));
    for (int w = 0; w < nw; ++w) {
        const kba_lidar_view& v = views[work[w]];
        memcpy(v.depth_out, depths.data() + plan.feat_off[w], sizeof(float) * (size_t)v.n_features);
    }
    return KBA_OK;
}

}  // namespace

extern "C" int kba_lidar_depth_batch(kba_handle* h, int32_t n_clouds, const kba_lidar_cloud* clouds, int32_t n_views,
                                     const kba_lidar_view* views, const kba_lidar_options* opt, float* device_ms) {
    return lidar_batch(h, n_clouds, clouds, n_views, views, opt, false, device_ms, "kba_lidar_depth_batch");
}

extern "C" int kba_lidar_depth_batch_opts(kba_handle* h, int32_t n_clouds, const kba_lidar_cloud* clouds, int32_t n_views,
                                          const kba_lidar_view* views, const kba_lidar_options* opts, float* device_ms) {
    return lidar_batch(h, n_clouds, clouds, n_views, views, opts, true, device_ms, "kba_lidar_depth_batch_opts");
}

// the one-view, one-cloud batch
extern "C" int kba_lidar_depth(kba_handle* h, const float* cloud, int32_t n_points, int32_t stride, const double* T,
                               const double* intr, const float* feats, int32_t n_feats, const kba_lidar_options* o,
                               float* depth_out, float* device_ms) {
    if (!h || !cloud || !T || !intr || !feats || !o || !depth_out || stride < 3 || n_points < 0 || n_feats < 0)
        return kba_internal_fail(KBA_ERR_BAD_ARG, "bad argument to kba_lidar_depth");
    const kba_lidar_cloud c{cloud, n_points, stride};
    const kba_lidar_view v{0, n_feats, T, intr, feats, depth_out};
    return lidar_batch(h, 1, &c, 1, &v, o, false, device_ms, "kba_lidar_depth");
}
