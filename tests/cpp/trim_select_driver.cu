// trim_select_driver.cu -- runs kba::trim_select_group (kba_controller.cuh), the quantile trimming of one residual group, in
// one CTA on cases read from a file, so tests/test_trim_select.py can hold its decisions to an exact-rank reference.
//
//   trim_select_driver <cases.bin> <masks.bin>
//
// cases.bin (little-endian): int32 n_sets, then per set
//   int32 n; double value[n]; int32 oid[n]; int32 n_runs; n_runs x { int32 block, int32 min_groups, double quantile }
// masks.bin: per set and run, in input order: float ms (the kernel's time), uint8 rejected[n]
//
// Each run selects twice in a row on the same shared state, as the solver kernels do with their residual groups; the second
// selection of the same group must not change the mask.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "kba_controller.cuh"

#define CK(x)                                                                                   \
    do {                                                                                        \
        cudaError_t e_ = (x);                                                                   \
        if (e_ != cudaSuccess) {                                                                \
            fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); \
            exit(2);                                                                            \
        }                                                                                       \
    } while (0)

__global__ void k_trim(const double* v, const int* oid, int n, double quant, int min_groups, uint8_t* rej) {
    __shared__ kba::TrimSmem sm;
    for (int j = threadIdx.x; j < n; j += blockDim.x) rej[j] = 0;
    __syncthreads();
    for (int rep = 0; rep < 2; ++rep)
        kba::trim_select_group(sm, n, quant, min_groups, [v](int j) { return v[j]; }, [oid](int j) { return oid[j]; }, rej);
}

template <typename T>
static void take(FILE* f, T* p, size_t n) {
    if (n && fread(p, sizeof(T), n, f) != n) { fprintf(stderr, "truncated case file\n"); exit(2); }
}

int main(int argc, char** argv) {
    if (argc != 3) { fprintf(stderr, "usage: %s cases.bin masks.bin\n", argv[0]); return 2; }
    FILE* in = fopen(argv[1], "rb");
    FILE* out = fopen(argv[2], "wb");
    if (!in || !out) { fprintf(stderr, "cannot open the case or mask file\n"); return 2; }
    int n_sets = 0;
    take(in, &n_sets, 1);
    cudaEvent_t a, b;
    CK(cudaEventCreate(&a));
    CK(cudaEventCreate(&b));
    for (int s = 0; s < n_sets; ++s) {
        int n = 0, n_runs = 0;
        take(in, &n, 1);
        std::vector<double> v(n);
        std::vector<int> oid(n);
        take(in, v.data(), n);
        take(in, oid.data(), n);
        take(in, &n_runs, 1);
        double* d_v = nullptr;
        int* d_oid = nullptr;
        uint8_t* d_rej = nullptr;
        const size_t m = n > 0 ? (size_t)n : 1;
        CK(cudaMalloc(&d_v, m * sizeof(double)));
        CK(cudaMalloc(&d_oid, m * sizeof(int)));
        CK(cudaMalloc(&d_rej, m));
        CK(cudaMemcpy(d_v, v.data(), (size_t)n * sizeof(double), cudaMemcpyHostToDevice));
        CK(cudaMemcpy(d_oid, oid.data(), (size_t)n * sizeof(int), cudaMemcpyHostToDevice));
        std::vector<uint8_t> rej(m);
        double ms_set = 0.0;
        for (int r = 0; r < n_runs; ++r) {
            int block = 0, min_groups = 0;
            double quant = 0.0;
            take(in, &block, 1);
            take(in, &min_groups, 1);
            take(in, &quant, 1);
            if (block < 32 || block > 512 || block % 32) { fprintf(stderr, "block %d: a multiple of 32 up to 512\n", block); return 2; }
            CK(cudaEventRecord(a));
            k_trim<<<1, block>>>(d_v, d_oid, n, quant, min_groups, d_rej);
            CK(cudaEventRecord(b));
            CK(cudaGetLastError());
            CK(cudaEventSynchronize(b));
            float ms = 0.f;
            CK(cudaEventElapsedTime(&ms, a, b));
            ms_set += ms;
            CK(cudaMemcpy(rej.data(), d_rej, (size_t)n, cudaMemcpyDeviceToHost));
            fwrite(&ms, sizeof ms, 1, out);
            fwrite(rej.data(), 1, (size_t)n, out);
        }
        CK(cudaFree(d_v));
        CK(cudaFree(d_oid));
        CK(cudaFree(d_rej));
        if (getenv("TRIM_DRIVER_PROGRESS")) { fprintf(stderr, "set %d: %d items, %d runs, %.3f ms\n", s, n, n_runs, ms_set); fflush(stderr); }
    }
    fclose(in);
    if (fclose(out) != 0) { fprintf(stderr, "cannot write the mask file\n"); return 2; }
    return 0;
}
