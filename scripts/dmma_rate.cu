// dmma_rate.cu -- issue rate of the FP64 tensor-core shapes of sm_90 (mma.sync m8n8k4, m16n8k4, m16n8k8, m16n8k16), and a
// check of the fragment layouts the Schur kernel relies on (PTX ISA, "Matrix fragments for mma.m16n8k*", .f64).
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o dmma_rate scripts/dmma_rate.cu && ./dmma_rate
//
// Rate: one CTA per SM, 4 or 8 warps per SM sub-partition, each warp with 4 independent accumulators (2 for m16n8k16;
// latency hidden by the other warps as well).  Cycles from clock64() (CTA-wide, between two barriers), wall time from CUDA events.
#include <cuda_runtime.h>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

template <int M, int K> struct Shape;
template <> struct Shape<8, 4> { static constexpr int na = 1, nb = 1, nc = 2; static constexpr const char* name = "m8n8k4"; };
template <> struct Shape<16, 4> { static constexpr int na = 2, nb = 1, nc = 4; static constexpr const char* name = "m16n8k4"; };
template <> struct Shape<16, 8> { static constexpr int na = 4, nb = 2, nc = 4; static constexpr const char* name = "m16n8k8"; };
template <> struct Shape<16, 16> { static constexpr int na = 8, nb = 4, nc = 4; static constexpr const char* name = "m16n8k16"; };

template <int M, int K>
__device__ __forceinline__ void mma(double* c, const double* a, const double* b);
template <> __device__ __forceinline__ void mma<8, 4>(double* c, const double* a, const double* b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c[0]), "+d"(c[1]) : "d"(a[0]), "d"(b[0]));
}
template <> __device__ __forceinline__ void mma<16, 4>(double* c, const double* a, const double* b) {
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(b[0]));
}
template <> __device__ __forceinline__ void mma<16, 8>(double* c, const double* a, const double* b) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
}
template <> __device__ __forceinline__ void mma<16, 16>(double* c, const double* a, const double* b) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, {%0,%1,%2,%3};"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

constexpr int kUnroll = 8;
// independent accumulators per warp: m16n8k16 keeps 2 so that its fragments fit 64 registers at 1024 threads
template <int M, int K> __host__ __device__ constexpr int acc_count() { return K == 16 ? 2 : 4; }

template <int M, int K>
__global__ void __launch_bounds__(1024, 1) k_rate(double* out, const double* in, int iters, long long* cycles) {
    using S = Shape<M, K>;
    constexpr int kAcc = acc_count<M, K>();
    double a[S::na], b[S::nb], c[kAcc][S::nc];
    for (int i = 0; i < S::na; ++i) a[i] = in[(threadIdx.x + 7 * i) & 255];
    for (int i = 0; i < S::nb; ++i) b[i] = in[(threadIdx.x + 13 * i + 3) & 255];
    for (int j = 0; j < kAcc; ++j)
        for (int i = 0; i < S::nc; ++i) c[j][i] = 0.0;
    __syncthreads();
    const long long t0 = clock64();
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int u = 0; u < kUnroll; ++u)
#pragma unroll
            for (int j = 0; j < kAcc; ++j) mma<M, K>(c[j], a, b);
    }
    __syncthreads();
    const long long t1 = clock64();
    double s = 0.0;
    for (int j = 0; j < kAcc; ++j)
        for (int i = 0; i < S::nc; ++i) s += c[j][i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

// D = A B for one warp with the fragment layouts of the PTX ISA (A row-major M x K, B column-major K x 8, D M x 8)
template <int M, int K>
__global__ void k_layout(double* d, const double* A, const double* B) {
    using S = Shape<M, K>;
    const int lane = threadIdx.x, g = lane >> 2, t = lane & 3;
    double a[S::na], b[S::nb], c[S::nc];
    for (int i = 0; i < S::na; ++i) a[i] = A[(g + 8 * (i & 1) * (M == 16)) * K + t + 4 * (M == 16 ? i >> 1 : i)];
    for (int i = 0; i < S::nb; ++i) b[i] = B[g * K + t + 4 * i];
    for (int i = 0; i < S::nc; ++i) c[i] = 0.0;
    mma<M, K>(c, a, b);
    for (int i = 0; i < S::nc; ++i) d[(g + 8 * (i >> 1)) * 8 + 2 * t + (i & 1)] = c[i];
}

template <int M, int K>
void run(int sms, int clock_khz) {
    using S = Shape<M, K>;
    // layout check against the host product
    std::vector<double> A(M * K), B(8 * K), D(M * 8);
    for (int i = 0; i < M * K; ++i) A[i] = 1.0 + (i * 37 % 101) / 64.0;
    for (int i = 0; i < 8 * K; ++i) B[i] = -2.0 + (i * 53 % 97) / 32.0;
    double *dA, *dB, *dD;
    CK(cudaMalloc(&dA, A.size() * 8)); CK(cudaMalloc(&dB, B.size() * 8)); CK(cudaMalloc(&dD, D.size() * 8));
    CK(cudaMemcpy(dA, A.data(), A.size() * 8, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dB, B.data(), B.size() * 8, cudaMemcpyHostToDevice));
    k_layout<M, K><<<1, 32>>>(dD, dA, dB);
    CK(cudaGetLastError());
    CK(cudaMemcpy(D.data(), dD, D.size() * 8, cudaMemcpyDeviceToHost));
    double err = 0.0;
    for (int i = 0; i < M; ++i)
        for (int j = 0; j < 8; ++j) {
            double r = 0.0;
            for (int k = 0; k < K; ++k) r += A[i * K + k] * B[j * K + k];
            err = fmax(err, fabs(D[i * 8 + j] - r) / fmax(1.0, fabs(r)));
        }
    CK(cudaFree(dA)); CK(cudaFree(dB)); CK(cudaFree(dD));
    printf("%-9s layout check: max rel error %.1e %s\n", S::name, err, err < 1e-14 ? "ok" : "MISMATCH");

    double *in, *out;
    long long* cyc;
    CK(cudaMalloc(&in, 256 * 8)); CK(cudaMemset(in, 0, 256 * 8));
    CK(cudaMalloc(&out, (size_t)sms * 1024 * 8)); CK(cudaMalloc(&cyc, sms * 8));
    std::vector<long long> hc(sms);
    for (int wps : {4, 8}) {
        const int threads = 32 * 4 * wps, iters = 4096;
        k_rate<M, K><<<sms, threads>>>(out, in, 64, cyc);  // warm-up
        CK(cudaGetLastError());
        cudaEvent_t e0, e1;
        CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
        CK(cudaEventRecord(e0));
        k_rate<M, K><<<sms, threads>>>(out, in, iters, cyc);
        CK(cudaGetLastError());
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        float ms = 0.f;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        CK(cudaMemcpy(hc.data(), cyc, sms * 8, cudaMemcpyDeviceToHost));
        long long cmax = 0;
        for (long long c : hc) cmax = c > cmax ? c : cmax;
        const double per_sm = (double)(threads / 32) * iters * kUnroll * acc_count<M, K>();  // MMAs per SM
        const double flop = 2.0 * M * 8 * K;
        printf("%-9s %d warps/SMSP: %.3f MMA/clk/SM = %.1f FP64 FLOP/clk/SM; %.2f ms wall, %.1f TFLOP/s (%d SMs)", S::name, wps,
               per_sm / cmax, per_sm * flop / cmax, ms, per_sm * sms * flop / (ms * 1e-3) / 1e12, sms);
        if (clock_khz > 0) printf(", %.0f MHz effective", cmax / (ms * 1e-3) / 1e6);
        printf("\n");
        CK(cudaEventDestroy(e0)); CK(cudaEventDestroy(e1));
    }
    CK(cudaFree(in)); CK(cudaFree(out)); CK(cudaFree(cyc));
}

int main() {
    cudaDeviceProp p;
    CK(cudaGetDeviceProperties(&p, 0));
    int clk = 0;
    cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
    printf("%s, %d SMs, sm_%d%d, max SM clock %d MHz\n", p.name, p.multiProcessorCount, p.major, p.minor, clk / 1000);
    fflush(stdout);
    if (std::system("nvidia-smi --query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks_throttle_reasons.active --format=csv")) printf("nvidia-smi failed\n");
    run<8, 4>(p.multiProcessorCount, clk);
    run<16, 4>(p.multiProcessorCount, clk);
    run<16, 8>(p.multiProcessorCount, clk);
    run<16, 16>(p.multiProcessorCount, clk);
    if (std::system("nvidia-smi --query-gpu=clocks.sm,power.draw,clocks_throttle_reasons.active --format=csv")) printf("nvidia-smi failed\n");
    return 0;
}
