// W ranks of the virtual-node exchange in one cooperative launch on one GPU (include/distegnn_b200_testing_comm.h).  The
// device code is the product's: comm_slot_allreduce (comm.cuh) and the update fragment (virtual_update_graph.cuh);
// build.py links comm.cu and virtual_update.cu into this library too, so the communicators are the product's.
#include <string.h>

#include "../../../include/distegnn_b200_testing_comm.h"
#include "common.cuh"
#include "virtual_update.cuh"

namespace degnn {
namespace {

#define RANKS_CUDA_TRY(expr)                                                                       \
    do {                                                                                           \
        cudaError_t e__ = (expr);                                                                  \
        if (e__ != cudaSuccess) {                                                                  \
            ::degnn::set_error("%s: %s failed: %s", __func__, #expr, cudaGetErrorString(e__));     \
            (void)cudaGetLastError();                                                              \
            return DISTEGNN_ECUDA;                                                                 \
        }                                                                                          \
    } while (0)

constexpr int PACKED_THREADS = 256;     // allreduce_packed_kernel's block

struct PauseSpec {
    unsigned long long max_ns;
    unsigned long long seed;
    int schedule;
};

// A pause of the calling thread, a function of (seed, rank, slot, call) only, so every thread of the CTA waits as long.
struct SeededPause {
    PauseSpec p;
    int rank, slot, call, world;
    __device__ __forceinline__ void operator()() const {
        unsigned long long ns = 0;
        if (p.schedule == DISTEGNN_PAUSE_ONE_SLOW_RANK) {
            ns = rank == (int)((p.seed + (unsigned long long)call) % (unsigned long long)world) ? p.max_ns : 0ull;
        } else if (p.max_ns) {
            unsigned long long h = p.seed ^ 0x9e3779b97f4a7c15ull;       // splitmix64 over the four indices
            for (unsigned long long v : {(unsigned long long)rank, (unsigned long long)slot, (unsigned long long)call}) {
                h += v + 0x9e3779b97f4a7c15ull;
                h = (h ^ (h >> 30)) * 0xbf58476d1ce4e5b9ull;
                h = (h ^ (h >> 27)) * 0x94d049bb133111ebull;
                h ^= h >> 31;
            }
            ns = h % (p.max_ns + 1);
        }
        if (!ns) return;
        const unsigned long long t0 = globaltimer_ns();
        while (globaltimer_ns() - t0 < ns) {
        }
    }
};

// Per-rank arguments of the twins, in one device block per launch.
struct PackedRanks {
    CommDev cds[COMM_MAX_WORLD];
    float* bufs[COMM_MAX_WORLD];
};
struct UpdateRanks {
    CommDev cds[COMM_MAX_WORLD];
    VUpdArgs as[COMM_MAX_WORLD];
};

__global__ void __launch_bounds__(PACKED_THREADS)
    allreduce_packed_ranks_kernel(const PackedRanks* ra, int64_t count, int calls, PauseSpec ps) {
    const int slot = blockIdx.x, r = blockIdx.y;
    const CommDev& cd = ra->cds[r];
    float* const* bufs = ra->bufs;
    const int64_t o = (int64_t)slot * cd.stride;
    const int n = (int)min((int64_t)cd.stride, count - o);
    for (int c = 0; c < calls; ++c)
        comm_slot_allreduce(cd, slot, bufs[r] + (int64_t)c * count + o, n, SeededPause{ps, r, slot, c, cd.world});
}

__global__ void __launch_bounds__(VU_THREADS)
    virtual_update_ranks_kernel(const UpdateRanks* ra, PauseSpec ps) {
    constexpr bool SYNC = true;
    const int b = blockIdx.x, r = blockIdx.y;
    const VUpdArgs& a = ra->as[r];
    const CommDev& cd = ra->cds[r];
    const SeededPause pause{ps, r, b, 0, cd.world};
#include "virtual_update_graph.cuh"
}

// The communicators of ranks 0..world-1 in rank order, connected, with capacity for `slots` slots of `floats` floats.
int ranks_of(const char* who, void* const* comms, int world, int64_t slots, int64_t floats, CommDev* cds) {
    if (!comms) { set_error("%s: null comms", who); return DISTEGNN_EINVAL; }
    if (world < 1 || world > COMM_MAX_WORLD) { set_error("%s: world %d outside [1,16]", who, world); return DISTEGNN_EINVAL; }
    int dev = -1;
    RANKS_CUDA_TRY(cudaGetDevice(&dev));
    for (int r = 0; r < world; ++r) {
        const CommHost* c = (const CommHost*)comms[r];
        if (!c) { set_error("%s: null communicator of rank %d", who, r); return DISTEGNN_EINVAL; }
        if (!c->connected || c->dev.world != world || c->dev.rank != r || c->device != dev) {
            set_error("%s: comms[%d] is not the connected rank %d of a world of %d on the current device", who, r, r, world);
            return DISTEGNN_EINVAL;
        }
        if (slots > c->dev.max_slots || floats > c->dev.stride) {
            set_error("%s: %lld slots of %lld floats exceed the capacity (%d slots of %d floats)", who, (long long)slots,
                      (long long)floats, c->dev.max_slots, c->dev.stride);
            return DISTEGNN_EINVAL;
        }
        cds[r] = c->dev;
    }
    return DISTEGNN_OK;
}

int device_ctas(const void* kernel, int threads, int* out) {
    int dev = 0, sms = 0, per_sm = 0;
    RANKS_CUDA_TRY(cudaGetDevice(&dev));
    RANKS_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    RANKS_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, 0));
    *out = per_sm * sms;
    return DISTEGNN_OK;
}

// Copies the per-rank arguments `host_block` to a stream-ordered device block whose address goes to *block (the kernel's
// first parameter, params[0] == block), launches `kernel` cooperatively on an (x, world) grid if all of its CTAs fit on
// the device at once, and frees the block behind the launch.
int launch_ranks(const char* who, const void* kernel, int threads, int64_t x, int world, const void* host_block,
                 size_t bytes, void** block, void** params, cudaStream_t stream) {
    int fit = 0;
    if (int rc = device_ctas(kernel, threads, &fit)) return rc;
    if (x * world > fit) {
        set_error("%s: %lld x %d CTAs do not fit on the device at once (at most %d co-resident CTAs)", who, (long long)x,
                  world, fit);
        return DISTEGNN_EINVAL;
    }
    RANKS_CUDA_TRY(cudaMallocAsync(block, bytes, stream));
    cudaError_t e = cudaMemcpyAsync(*block, host_block, bytes, cudaMemcpyHostToDevice, stream);
    if (e == cudaSuccess) e = cudaLaunchCooperativeKernel(kernel, dim3((unsigned)x, (unsigned)world), dim3(threads), params, 0,
                                                          stream);
    const cudaError_t f = cudaFreeAsync(*block, stream);
    if (e == cudaSuccess) e = f;
    if (e != cudaSuccess) {
        set_error("%s: %s", who, cudaGetErrorString(e));
        (void)cudaGetLastError();
        return DISTEGNN_ECUDA;
    }
    return DISTEGNN_OK;
}

}  // namespace
}  // namespace degnn

using namespace degnn;

extern "C" {

int distegnn_comm_connect_local(void* const* comms, int world) {
    DEGNN_CHECK_ARG(comms, "null comms");
    DEGNN_CHECK_ARG(world >= 1 && world <= COMM_MAX_WORLD, "world size outside [1,16]");
    CommHost* by_rank[COMM_MAX_WORLD] = {};
    for (int i = 0; i < world; ++i) {
        CommHost* c = (CommHost*)comms[i];
        DEGNN_CHECK_ARG(c, "null communicator");
        DEGNN_CHECK_ARG(!c->connected, "communicator already connected");
        DEGNN_CHECK_ARG(c->dev.world == world, "communicator made for another world size");
        DEGNN_CHECK_ARG(!by_rank[c->dev.rank], "duplicate rank");
        by_rank[c->dev.rank] = c;
    }
    for (int r = 0; r < world; ++r) DEGNN_CHECK_ARG(by_rank[r], "missing rank");
    const CommHost* c0 = by_rank[0];
    for (int r = 1; r < world; ++r) {
        DEGNN_CHECK_ARG(by_rank[r]->dev.max_slots == c0->dev.max_slots, "unequal max_slots");
        DEGNN_CHECK_ARG(by_rank[r]->dev.stride == c0->dev.stride, "unequal slot stride");
        DEGNN_CHECK_ARG(by_rank[r]->device == c0->device, "communicators on different devices");
    }
    const SegLayout s = seg_layout(world, c0->dev.max_slots, c0->dev.stride);
    for (int i = 0; i < world; ++i) {
        CommHost* c = by_rank[i];
        for (int r = 0; r < world; ++r) {
            c->peer_base[r] = nullptr;          // nothing for distegnn_comm_destroy to unmap
            c->dev.flags[r] = (unsigned*)((char*)by_rank[r]->segment + s.flags_off);
            c->dev.data[r] = (float*)((char*)by_rank[r]->segment + s.data_off);
        }
        c->dev.epoch = (unsigned*)((char*)c->segment + s.epoch_off);
        c->dev.status = (unsigned*)((char*)c->segment + s.status_off);
        c->connected = true;
    }
    return DISTEGNN_OK;
}

int distegnn_comm_ranks_capacity(int* packed_ctas, int* update_ctas) {
    DEGNN_CHECK_ARG(packed_ctas && update_ctas, "null pointer");
    if (int rc = device_ctas((const void*)allreduce_packed_ranks_kernel, PACKED_THREADS, packed_ctas)) return rc;
    return device_ctas((const void*)virtual_update_ranks_kernel, VU_THREADS, update_ctas);
}

int distegnn_allreduce_packed_ranks(void* const* comms, int world, float* const* bufs, int64_t count, int calls,
                                    int schedule, int64_t max_pause_ns, uint64_t seed, void* stream) {
    DEGNN_CHECK_ARG(comms && bufs, "null pointer");
    DEGNN_CHECK_ARG(world >= 1 && world <= COMM_MAX_WORLD, "world size outside [1,16]");
    DEGNN_CHECK_ARG(count >= 0 && calls >= 0, "negative count or calls");
    DEGNN_CHECK_ARG(max_pause_ns >= 0, "negative pause");
    DEGNN_CHECK_ARG(schedule == DISTEGNN_PAUSE_SEEDED || schedule == DISTEGNN_PAUSE_ONE_SLOW_RANK, "unknown pause schedule");
    for (int r = 0; r < world; ++r) DEGNN_CHECK_ARG(bufs[r], "null buffer");
    if (count == 0 || calls == 0) return DISTEGNN_OK;
    const CommHost* c0 = (const CommHost*)comms[0];
    DEGNN_CHECK_ARG(c0, "null communicator of rank 0");
    const int64_t slots = (count + c0->dev.stride - 1) / c0->dev.stride;   // every stride is checked against rank 0's
    PackedRanks host;
    memset(&host, 0, sizeof(host));
    if (int rc = ranks_of(__func__, comms, world, slots, c0->dev.stride, host.cds)) return rc;
    for (int r = 0; r < world; ++r) {
        DEGNN_CHECK_ARG(host.cds[r].stride == c0->dev.stride, "unequal slot stride");
        host.bufs[r] = bufs[r];
    }
    void* block = nullptr;
    PauseSpec ps{(unsigned long long)max_pause_ns, (unsigned long long)seed, schedule};
    void* params[] = {&block, &count, &calls, &ps};
    return launch_ranks(__func__, (const void*)allreduce_packed_ranks_kernel, PACKED_THREADS, slots, world, &host,
                        sizeof(host), &block, params, (cudaStream_t)stream);
}

int distegnn_virtual_update_fwd_ranks(void* const* comms, int world, int n_graphs, int A, int C, int Na, unsigned flags,
                                      float* const* vsum, float* const* Xv, float* const* Hv, const float* layer_params,
                                      const float* next_layer_params, float* const* G, const float* init_loc_mean,
                                      const float* init_hv0, int64_t max_pause_ns, uint64_t seed, void* stream) {
    DEGNN_CHECK_ARG(comms && vsum && Xv, "null pointer");
    DEGNN_CHECK_ARG(world >= 1 && world <= COMM_MAX_WORLD, "world size outside [1,16]");
    DEGNN_CHECK_ARG(max_pause_ns >= 0, "negative pause");
    if (int rc = check_dims(A, C, Na)) return rc;
    if (n_graphs == 0) return DISTEGNN_OK;
    UpdateRanks host;
    memset(&host, 0, sizeof(host));
    for (int r = 0; r < world; ++r)
        if (int rc = virtual_update_args(__func__, n_graphs, A, C, Na, flags, vsum[r], Xv[r], Hv ? Hv[r] : nullptr,
                                         layer_params, next_layer_params, G ? G[r] : nullptr, init_loc_mean, init_hv0,
                                         &host.as[r]))
            return rc;
    if (int rc = ranks_of(__func__, comms, world, n_graphs, host.as[0].K, host.cds)) return rc;
    void* block = nullptr;
    PauseSpec ps{(unsigned long long)max_pause_ns, (unsigned long long)seed, DISTEGNN_PAUSE_SEEDED};
    void* params[] = {&block, &ps};
    return launch_ranks(__func__, (const void*)virtual_update_ranks_kernel, VU_THREADS, n_graphs, world, &host,
                        sizeof(host), &block, params, (cudaStream_t)stream);
}

}  // extern "C"
