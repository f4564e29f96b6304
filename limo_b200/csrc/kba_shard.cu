// kba_shard.cu -- exchange plumbing of the sharded window solve (include/kba_b200.h, "ONE large window sharded ...").
// Two kinds of communicator plug into kba::Exchange:
//   - NCCL, one process per GPU.  libnccl is opened at run time (dlopen) so that single-GPU users need no NCCL, and so that
//     inside a PyTorch process the library torch already loaded is the one used;
//   - in process: W handles of one process on ONE device, each rank solved from its own host thread (kba_shard_comm_create_local).
//     It lets one GPU run and check the cross-rank sums of a W-rank solve, which NCCL refuses (two ranks on one device).
#include <dlfcn.h>

#include <condition_variable>
#include <cstdio>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>

#include <cuda_runtime.h>
#include <nccl.h>  // types only: no symbol of libnccl is linked

#include "kba_b200.h"
#include "kba_kernels.h"

extern "C" {
int kba_internal_stream(kba_handle* h, cudaStream_t* s, int* device);
int kba_internal_fail(int code, const char* msg);
}

namespace {

struct NcclApi {
    void* lib = nullptr;
    decltype(&ncclGetUniqueId) get_unique_id = nullptr;
    decltype(&ncclCommInitRank) comm_init_rank = nullptr;
    decltype(&ncclAllReduce) all_reduce = nullptr;
    decltype(&ncclCommDestroy) comm_destroy = nullptr;
    decltype(&ncclGetErrorString) error_string = nullptr;
    bool ok() const { return lib && get_unique_id && comm_init_rank && all_reduce && comm_destroy && error_string; }
};

NcclApi& api() {
    static NcclApi a;
    if (a.lib) return a;
    for (const char* name : {"libnccl.so.2", "libnccl.so"}) {
        a.lib = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
        if (a.lib) break;
    }
    if (!a.lib) return a;
    a.get_unique_id = (decltype(a.get_unique_id))dlsym(a.lib, "ncclGetUniqueId");
    a.comm_init_rank = (decltype(a.comm_init_rank))dlsym(a.lib, "ncclCommInitRank");
    a.all_reduce = (decltype(a.all_reduce))dlsym(a.lib, "ncclAllReduce");
    a.comm_destroy = (decltype(a.comm_destroy))dlsym(a.lib, "ncclCommDestroy");
    a.error_string = (decltype(a.error_string))dlsym(a.lib, "ncclGetErrorString");
    return a;
}

int nccl_fail(const char* what, ncclResult_t r) {
    std::string m = std::string(what) + ": " + (api().error_string ? api().error_string(r) : "nccl error");
    return kba_internal_fail(KBA_ERR_NCCL, m.c_str());
}

// ---- in-process exchange ------------------------------------------------------------------------------------------------
constexpr int kMaxLocalWorld = 16;

struct LocalSrc { const double* p[kMaxLocalWorld]; };

// out[i] = src_0[i] (+) src_1[i] (+) ... in rank order: every rank computes the same bits
__global__ void __launch_bounds__(256) k_local_reduce(LocalSrc src, int world, long long count, int op, double* out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    double v = src.p[0][i];
    for (int r = 1; r < world; ++r) v = op == 1 ? fmax(v, src.p[r][i]) : v + src.p[r][i];
    out[i] = v;
}

// State shared by the W ranks of one in-process communicator.  An all-reduce of rank r, called from r's host thread:
//   1. record `ready[r]` on r's stream (the send buffer is written), 2. host barrier, 3. r's stream waits for every `ready`,
//   4. r's reduce kernel reads the W send buffers in rank order, 5. record `done[r]`, host barrier, r's stream waits for every
//   `done`: no rank writes a send buffer again (nor, in place, its result) before every rank's kernel has read it.
// A rank that fails breaks the group: the barriers then release every waiting rank with an error, now and later.
struct LocalGroup {
    int world = 0, device = 0;
    std::mutex m;
    std::condition_variable cv;
    int arrived = 0;
    long long generation = 0;
    bool broken = false;
    std::string why;
    cudaEvent_t ready[kMaxLocalWorld] = {}, done[kMaxLocalWorld] = {};
    const double* send[kMaxLocalWorld] = {};
    long long count[kMaxLocalWorld] = {};
    int op[kMaxLocalWorld] = {};
    double* tmp[kMaxLocalWorld] = {};       // per rank: the sum of an in-place all-reduce before it is copied over its buffer
    long long tmp_cap[kMaxLocalWorld] = {};

    bool barrier() {
        std::unique_lock<std::mutex> lk(m);
        if (broken) return false;
        const long long gen = generation;
        if (++arrived == world) {
            arrived = 0;
            ++generation;
            cv.notify_all();
            return true;
        }
        cv.wait(lk, [&] { return broken || generation != gen; });
        return generation != gen;
    }
    void breakup(const std::string& msg) {
        std::lock_guard<std::mutex> lk(m);
        if (!broken) { broken = true; why = msg; }
        cv.notify_all();
    }
    std::string reason() {
        std::lock_guard<std::mutex> lk(m);
        return why;
    }
    ~LocalGroup() {
        cudaSetDevice(device);
        for (int r = 0; r < world; ++r) {
            if (ready[r]) cudaEventDestroy(ready[r]);
            if (done[r]) cudaEventDestroy(done[r]);
            if (tmp[r]) cudaFree(tmp[r]);
        }
    }
};

}  // namespace

struct kba_shard_comm {
    ncclComm_t comm = nullptr;                // NCCL kind
    std::shared_ptr<LocalGroup> local;        // in-process kind
    int rank = 0, world = 1, device = 0;
};

static int shard_allreduce(void* user, const double* send, double* recv, long long count, int op, cudaStream_t s) {
    kba_shard_comm* c = (kba_shard_comm*)user;
    const ncclResult_t r = api().all_reduce(send, recv, (size_t)count, ncclDouble, op == 1 ? ncclMax : ncclSum, c->comm, s);
    return r == ncclSuccess ? 0 : nccl_fail("ncclAllReduce", r);
}

static int local_fail(LocalGroup& g, const std::string& msg) {
    g.breakup(msg);
    return kba_internal_fail(KBA_ERR_NCCL, ("in-process exchange: " + g.reason()).c_str());
}

static int local_allreduce(void* user, const double* send, double* recv, long long count, int op, cudaStream_t s) {
    kba_shard_comm* c = (kba_shard_comm*)user;
    LocalGroup& g = *c->local;
    const int r = c->rank, W = g.world;
    const bool in_place = send == recv;
    if (in_place && g.tmp_cap[r] < count) {  // grows once per size; the first solve of a batch meets every size
        if (g.tmp[r]) cudaFree(g.tmp[r]);
        g.tmp[r] = nullptr; g.tmp_cap[r] = 0;
        if (cudaMalloc(&g.tmp[r], (size_t)count * sizeof(double)) != cudaSuccess) return local_fail(g, "out of device memory");
        g.tmp_cap[r] = count;
    }
    g.send[r] = send; g.count[r] = count; g.op[r] = op;
    if (cudaEventRecord(g.ready[r], s) != cudaSuccess) return local_fail(g, "cudaEventRecord failed");
    if (!g.barrier()) return local_fail(g, "another rank failed");
    LocalSrc src{};
    for (int q = 0; q < W; ++q) {
        if (g.count[q] != count || g.op[q] != op) return local_fail(g, "the ranks issued different all-reduces");
        src.p[q] = g.send[q];
        if (q != r && cudaStreamWaitEvent(s, g.ready[q], 0) != cudaSuccess) return local_fail(g, "cudaStreamWaitEvent failed");
    }
    double* out = in_place ? g.tmp[r] : recv;
    if (count > 0) k_local_reduce<<<(unsigned)((count + 255) / 256), 256, 0, s>>>(src, W, count, op, out);
    if (cudaGetLastError() != cudaSuccess || cudaEventRecord(g.done[r], s) != cudaSuccess) return local_fail(g, "reduce launch failed");
    if (!g.barrier()) return local_fail(g, "another rank failed");
    for (int q = 0; q < W; ++q)
        if (q != r && cudaStreamWaitEvent(s, g.done[q], 0) != cudaSuccess) return local_fail(g, "cudaStreamWaitEvent failed");
    if (in_place && count > 0 && cudaMemcpyAsync(recv, out, (size_t)count * sizeof(double), cudaMemcpyDeviceToDevice, s) != cudaSuccess)
        return local_fail(g, "cudaMemcpyAsync failed");
    return 0;
}

static void local_abort(void* user) { ((kba_shard_comm*)user)->local->breakup("a rank left the collective on an error"); }

// used by kba_api.cu
kba::Exchange kba_shard_exchange(kba_shard_comm* c) {
    kba::Exchange x;
    if (c->local) {
        x.allreduce = &local_allreduce;
        x.abort = &local_abort;
        x.capturable = false;  // host barriers at enqueue time
    } else {
        x.allreduce = &shard_allreduce;
    }
    x.user = c;
    x.rank = c->rank; x.world = c->world;
    return x;
}

extern "C" {

int kba_shard_unique_id(void* id_out) {
    static_assert(sizeof(ncclUniqueId) == KBA_SHARD_ID_BYTES, "NCCL unique id size");
    if (!id_out) return kba_internal_fail(KBA_ERR_BAD_ARG, "null id buffer");
    if (!api().ok()) return kba_internal_fail(KBA_ERR_NCCL, "libnccl.so.2 not found");
    ncclUniqueId id;
    const ncclResult_t r = api().get_unique_id(&id);
    if (r != ncclSuccess) return nccl_fail("ncclGetUniqueId", r);
    memcpy(id_out, &id, sizeof id);
    return KBA_OK;
}

int kba_shard_comm_create(kba_handle* h, int32_t rank, int32_t world, const void* id, kba_shard_comm** out) {
    if (!h || !id || !out || world < 1 || rank < 0 || rank >= world) return kba_internal_fail(KBA_ERR_BAD_ARG, "bad argument to kba_shard_comm_create");
    if (!api().ok()) return kba_internal_fail(KBA_ERR_NCCL, "libnccl.so.2 not found");
    cudaStream_t s;
    int device = 0;
    if (int rc = kba_internal_stream(h, &s, &device)) return rc;
    if (cudaSetDevice(device) != cudaSuccess) return kba_internal_fail(KBA_ERR_CUDA, "cudaSetDevice failed");
    kba_shard_comm* c = new kba_shard_comm;
    c->rank = rank; c->world = world; c->device = device;
    ncclUniqueId uid;
    memcpy(&uid, id, sizeof uid);
    const ncclResult_t r = api().comm_init_rank(&c->comm, world, uid, rank);
    if (r != ncclSuccess) { delete c; return nccl_fail("ncclCommInitRank", r); }
    *out = c;
    return KBA_OK;
}

int kba_shard_comm_create_local(kba_handle* const* handles, int32_t world, kba_shard_comm** out) {
    if (!handles || !out || world < 1 || world > kMaxLocalWorld)
        return kba_internal_fail(KBA_ERR_BAD_ARG, "bad argument to kba_shard_comm_create_local (1 <= world <= 16)");
    auto g = std::make_shared<LocalGroup>();
    g->world = world;
    for (int r = 0; r < world; ++r) {
        cudaStream_t s;
        int device = 0;
        if (int rc = kba_internal_stream(handles[r], &s, &device)) return rc;
        if (r == 0) g->device = device;
        if (device != g->device) return kba_internal_fail(KBA_ERR_BAD_ARG, "kba_shard_comm_create_local: the handles are on different devices");
        for (int q = 0; q < r; ++q)
            if (handles[q] == handles[r]) return kba_internal_fail(KBA_ERR_BAD_ARG, "kba_shard_comm_create_local: one handle per rank");
    }
    if (cudaSetDevice(g->device) != cudaSuccess) return kba_internal_fail(KBA_ERR_CUDA, "cudaSetDevice failed");
    for (int r = 0; r < world; ++r)
        if (cudaEventCreateWithFlags(&g->ready[r], cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&g->done[r], cudaEventDisableTiming) != cudaSuccess)
            return kba_internal_fail(KBA_ERR_CUDA, "cudaEventCreate failed");
    for (int r = 0; r < world; ++r) {
        kba_shard_comm* c = new kba_shard_comm;
        c->local = g;
        c->rank = r; c->world = world; c->device = g->device;
        out[r] = c;
    }
    return KBA_OK;
}

void kba_shard_comm_destroy(kba_shard_comm* c) {
    if (!c) return;
    if (c->comm && api().ok()) api().comm_destroy(c->comm);
    delete c;
}

}  // extern "C"
