// kba_lidar.cu -- lidar depth extraction on sm_90a (BASELINE config 4; C ABI: kba_lidar_depth in kba_b200.h).
//   k_lidar_bin<false>: project the cloud (coalesced float loads), count points per 16x16-pixel image cell
//   k_lidar_scan      : exclusive scan of the cell counts (one CTA)
//   k_lidar_bin<true> : project again and scatter (u, v, x, y, z, index) into cell-sorted order
//   k_lidar_feature   : one warp per feature: gather the pixel rectangle from the overlapping cells, depth histogram,
//                       largest triangle, plane / view-ray intersection, depth gates
// Compiled with -fmad=false: the arithmetic is single precision with the operation order of the specification so that the
// discrete decisions (rectangle membership, histogram bin, arg-max triangle) do not depend on FMA contraction.
#include <cstdint>
#include <string>

#include <cuda_runtime.h>

#include "kba_b200.h"

namespace {

constexpr int kCell = 16;      // pixels per cell side
constexpr int kMaxNb = 96;     // neighbours kept per feature
constexpr int kBins = 64;

struct LidarParams {
    float R[9], t[3], f, cx, cy;
    int width, height, cells_x, cells_y;
    float hw, hh, offx, offy, bw;
    int hist_min_count, min_points;
    float depth_min, depth_max, local_tol, crossnorm_min, viewray_min;
    int local_enabled;
};

struct ProjPt { float u, v, x, y, z; int idx; };

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

template <bool kFill>
__global__ void __launch_bounds__(256) k_lidar_bin(LidarParams P, const float* __restrict__ cloud, int n, int stride,
                                                   int* __restrict__ cell_count, const int* __restrict__ cell_start,
                                                   int* __restrict__ cell_cursor, ProjPt* __restrict__ sorted) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ProjPt q;
    if (!project(P, cloud + (size_t)i * stride, q)) return;
    const int cell = ((int)q.v / kCell) * P.cells_x + ((int)q.u / kCell);
    if (!kFill) {
        atomicAdd(&cell_count[cell], 1);
    } else {
        q.idx = i;
        sorted[cell_start[cell] + atomicAdd(&cell_cursor[cell], 1)] = q;
    }
}

__global__ void __launch_bounds__(1024) k_lidar_scan(const int* __restrict__ cnt, int* __restrict__ start, int ncell) {
    __shared__ int s_part[1024];
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

__global__ void __launch_bounds__(128) k_lidar_feature(LidarParams P, const ProjPt* __restrict__ sorted,
                                                       const int* __restrict__ cell_start, const float* __restrict__ feats,
                                                       int n_feats, float* __restrict__ out) {
    __shared__ ProjPt s_nb[4][kMaxNb];
    __shared__ int s_cnt[4][kBins];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int k = blockIdx.x * 4 + warp;
    if (k >= n_feats) return;
    ProjPt* nb = s_nb[warp];
    int* cnt = s_cnt[warp];
    const float fu = feats[2 * k], fv = feats[2 * k + 1];
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
    if (lane == 0) out[k] = result;
}

void quat_R(const double* q, float* R) {
    const double w = q[0], x = q[1], y = q[2], z = q[3];
    const double M[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y), 2 * (x * y + w * z), 1 - 2 * (x * x + z * z),
                         2 * (y * z - w * x), 2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)};
    for (int i = 0; i < 9; ++i) R[i] = (float)M[i];
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

extern "C" int kba_lidar_depth(kba_handle* h, const float* cloud, int32_t n_points, int32_t stride, const double* T,
                               const double* intr, const float* feats, int32_t n_feats, const kba_lidar_options* o,
                               float* depth_out, float* device_ms) {
    if (!h || !cloud || !T || !intr || !feats || !o || !depth_out || stride < 3 || n_points < 0 || n_feats < 0)
        return kba_internal_fail(KBA_ERR_BAD_ARG, "bad argument to kba_lidar_depth");
    cudaStream_t s;
    int device;
    if (kba_internal_stream(h, &s, &device) != KBA_OK) return KBA_ERR_BAD_ARG;
    LidarParams P;
    quat_R(T, P.R);
    P.t[0] = (float)T[4]; P.t[1] = (float)T[5]; P.t[2] = (float)T[6];
    P.f = (float)intr[0]; P.cx = (float)intr[1]; P.cy = (float)intr[2];
    P.width = o->image_width; P.height = o->image_height;
    P.cells_x = (P.width + kCell - 1) / kCell; P.cells_y = (P.height + kCell - 1) / kCell;
    P.hw = 0.5f * (float)o->rect_width; P.hh = 0.5f * (float)o->rect_height;
    P.offx = (float)o->rect_offset_x; P.offy = (float)o->rect_offset_y; P.bw = (float)o->hist_bin_width;
    P.hist_min_count = o->hist_min_count; P.min_points = o->min_points;
    P.depth_min = (float)o->depth_min; P.depth_max = (float)o->depth_max;
    P.local_enabled = o->local_rel_tolerance >= 0; P.local_tol = (float)o->local_rel_tolerance;
    P.crossnorm_min = (float)o->triangle_crossnorm_min; P.viewray_min = (float)o->viewray_plane_min;
    const int ncell = P.cells_x * P.cells_y;
    // one device workspace owned by the handle (grow-only): cloud | features | depths | cell counts, starts, cursors | sorted points
    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    const size_t b_cloud = al(sizeof(float) * (size_t)std::max(n_points, 1) * stride), b_feat = al(sizeof(float) * 2 * (size_t)std::max(n_feats, 1)),
                 b_out = al(sizeof(float) * (size_t)std::max(n_feats, 1)), b_cell = al(sizeof(int) * (size_t)(ncell + 1)),
                 b_sorted = al(sizeof(ProjPt) * (size_t)std::max(n_points, 1));
    void* ws = nullptr;
    if (kba_internal_workspace(h, b_cloud + b_feat + b_out + 3 * b_cell + b_sorted, &ws) != KBA_OK) return KBA_ERR_CUDA;
    char* wp = (char*)ws;
    float* d_cloud = (float*)wp; wp += b_cloud;
    float* d_feats = (float*)wp; wp += b_feat;
    float* d_out = (float*)wp; wp += b_out;
    int* d_cnt = (int*)wp; wp += b_cell;
    int* d_start = (int*)wp; wp += b_cell;
    int* d_cur = (int*)wp; wp += b_cell;
    ProjPt* d_sorted = (ProjPt*)wp;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    cudaError_t err = cudaSuccess;
    auto chk = [&](cudaError_t e) { if (err == cudaSuccess && e != cudaSuccess) err = e; };
    chk(cudaSetDevice(device));
    if (device_ms) { chk(cudaEventCreate(&e0)); chk(cudaEventCreate(&e1)); }
    if (err == cudaSuccess) {
        chk(cudaMemcpyAsync(d_cloud, cloud, sizeof(float) * (size_t)n_points * stride, cudaMemcpyHostToDevice, s));
        chk(cudaMemcpyAsync(d_feats, feats, sizeof(float) * 2 * (size_t)n_feats, cudaMemcpyHostToDevice, s));
        if (e0) chk(cudaEventRecord(e0, s));
        chk(cudaMemsetAsync(d_cnt, 0, sizeof(int) * ncell, s));
        chk(cudaMemsetAsync(d_cur, 0, sizeof(int) * ncell, s));
        const int gp = (n_points + 255) / 256;
        if (n_points > 0) k_lidar_bin<false><<<gp, 256, 0, s>>>(P, d_cloud, n_points, stride, d_cnt, nullptr, nullptr, nullptr);
        k_lidar_scan<<<1, 1024, 0, s>>>(d_cnt, d_start, ncell);
        if (n_points > 0) k_lidar_bin<true><<<gp, 256, 0, s>>>(P, d_cloud, n_points, stride, d_cnt, d_start, d_cur, d_sorted);
        if (n_feats > 0) k_lidar_feature<<<(n_feats + 3) / 4, 128, 0, s>>>(P, d_sorted, d_start, d_feats, n_feats, d_out);
        if (e1) chk(cudaEventRecord(e1, s));
        chk(cudaMemcpyAsync(depth_out, d_out, sizeof(float) * (size_t)n_feats, cudaMemcpyDeviceToHost, s));
        chk(cudaStreamSynchronize(s));
        chk(cudaGetLastError());
        if (err == cudaSuccess && device_ms) chk(cudaEventElapsedTime(device_ms, e0, e1));
    }
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
    if (err != cudaSuccess) return kba_internal_fail(KBA_ERR_CUDA, cudaGetErrorString(err));
    return KBA_OK;
}
