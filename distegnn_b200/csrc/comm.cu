// C ABI of the virtual-node sync (include/distegnn_b200.h, "collective" section): segment allocation + CUDA-IPC peer
// mapping on the host, and the stand-alone packed all-reduce kernel.  The fused all-reduce + virtual-node update lives in
// virtual_update.cu and uses the same device routine (comm.cuh).
#include <string.h>

#include "comm.cuh"
#include "common.cuh"

namespace degnn {

#define DEGNN_CUDA_TRY(expr)                                                                       \
    do {                                                                                           \
        cudaError_t e__ = (expr);                                                                  \
        if (e__ != cudaSuccess) {                                                                  \
            ::degnn::set_error("%s: %s failed: %s", __func__, #expr, cudaGetErrorString(e__));     \
            (void)cudaGetLastError();                                                              \
            return DISTEGNN_ECUDA;                                                                 \
        }                                                                                          \
    } while (0)

__global__ void __launch_bounds__(256) allreduce_packed_kernel(const CommDev cd, float* buf, int64_t count) {
    const int slot = blockIdx.x;
    const int64_t o = (int64_t)slot * cd.stride;
    const int n = (int)min((int64_t)cd.stride, count - o);
    comm_slot_allreduce(cd, slot, buf + o, n);
}

}  // namespace degnn

using namespace degnn;

extern "C" int distegnn_comm_handle_bytes(void) { return (int)sizeof(cudaIpcMemHandle_t); }

extern "C" int distegnn_comm_init(int rank, int world, int max_slots, int slot_floats, void** comm_out,
                                  void* handle_out_host) {
    DEGNN_CHECK_ARG(comm_out && handle_out_host, "null pointer");
    DEGNN_CHECK_ARG(world >= 1 && world <= COMM_MAX_WORLD, "world size outside [1,16]");
    DEGNN_CHECK_ARG(rank >= 0 && rank < world, "bad rank");
    DEGNN_CHECK_ARG(max_slots >= 1 && slot_floats >= 1, "bad capacity");
    CommHost* c = new CommHost();
    memset(c, 0, sizeof(*c));
    const int stride = (slot_floats + 3) / 4 * 4;
    const SegLayout s = seg_layout(world, max_slots, stride);
    DEGNN_CUDA_TRY(cudaGetDevice(&c->device));
    cudaError_t e = cudaMalloc(&c->segment, s.total);
    if (e != cudaSuccess) {
        set_error("distegnn_comm_init: cudaMalloc(%zu) failed: %s", s.total, cudaGetErrorString(e));
        delete c;
        return DISTEGNN_ECUDA;
    }
    c->segment_bytes = s.total;
    e = cudaMemset(c->segment, 0, s.total);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    cudaIpcMemHandle_t h;
    if (e == cudaSuccess) e = cudaIpcGetMemHandle(&h, c->segment);
    if (e != cudaSuccess) {
        set_error("distegnn_comm_init: %s", cudaGetErrorString(e));
        (void)cudaGetLastError();
        cudaFree(c->segment);
        delete c;
        return DISTEGNN_ECUDA;
    }
    memcpy(handle_out_host, &h, sizeof(h));
    c->dev.rank = rank;
    c->dev.world = world;
    c->dev.max_slots = max_slots;
    c->dev.stride = stride;
    c->dev.timeout_ns = 10ull * 1000ull * 1000ull * 1000ull;
    *comm_out = c;
    return DISTEGNN_OK;
}

extern "C" int distegnn_comm_connect(void* comm, const void* all_handles_host) {
    DEGNN_CHECK_ARG(comm && all_handles_host, "null pointer");
    CommHost* c = (CommHost*)comm;
    DEGNN_CHECK_ARG(!c->connected, "already connected");
    const SegLayout s = seg_layout(c->dev.world, c->dev.max_slots, c->dev.stride);
    const cudaIpcMemHandle_t* hs = (const cudaIpcMemHandle_t*)all_handles_host;
    for (int r = 0; r < c->dev.world; ++r) {
        void* base = c->segment;
        if (r != c->dev.rank) {
            cudaError_t e = cudaIpcOpenMemHandle(&base, hs[r], cudaIpcMemLazyEnablePeerAccess);
            if (e != cudaSuccess) {
                set_error("distegnn_comm_connect: cudaIpcOpenMemHandle(rank %d) failed: %s", r, cudaGetErrorString(e));
                (void)cudaGetLastError();
                for (int q = 0; q < r; ++q)
                    if (q != c->dev.rank && c->peer_base[q]) cudaIpcCloseMemHandle(c->peer_base[q]);
                memset(c->peer_base, 0, sizeof(c->peer_base));
                return DISTEGNN_ECUDA;
            }
        }
        c->peer_base[r] = base;
        c->dev.flags[r] = (unsigned*)((char*)base + s.flags_off);
        c->dev.data[r] = (float*)((char*)base + s.data_off);
    }
    c->dev.epoch = (unsigned*)((char*)c->segment + s.epoch_off);
    c->dev.status = (unsigned*)((char*)c->segment + s.status_off);
    c->connected = true;
    return DISTEGNN_OK;
}

extern "C" int distegnn_comm_set_timeout_ms(void* comm, int64_t ms) {
    DEGNN_CHECK_ARG(comm && ms > 0, "bad argument");
    ((CommHost*)comm)->dev.timeout_ns = (unsigned long long)ms * 1000000ull;
    return DISTEGNN_OK;
}

extern "C" int distegnn_comm_status(void* comm, int* status_host) {
    DEGNN_CHECK_ARG(comm && status_host, "null pointer");
    CommHost* c = (CommHost*)comm;
    DEGNN_CHECK_ARG(c->connected, "not connected");
    unsigned v = 0;
    DEGNN_CUDA_TRY(cudaMemcpy(&v, c->dev.status, sizeof(v), cudaMemcpyDeviceToHost));
    *status_host = (int)v;
    return DISTEGNN_OK;
}

// Unmap the peers' segments (this rank's own segment stays allocated: peers may still have it mapped).  Teardown order
// across ranks: everybody disconnects -> host barrier -> everybody destroys (CUDA leaves freeing an exported allocation
// that an importer still maps undefined).
extern "C" int distegnn_comm_disconnect(void* comm) {
    if (!comm) return DISTEGNN_OK;
    CommHost* c = (CommHost*)comm;
    for (int r = 0; r < c->dev.world; ++r)
        if (r != c->dev.rank && c->peer_base[r]) {
            cudaIpcCloseMemHandle(c->peer_base[r]);
            c->peer_base[r] = nullptr;
        }
    (void)cudaGetLastError();
    c->connected = false;
    return DISTEGNN_OK;
}

extern "C" int distegnn_comm_destroy(void* comm) {
    if (!comm) return DISTEGNN_OK;
    CommHost* c = (CommHost*)comm;
    for (int r = 0; r < c->dev.world; ++r)
        if (r != c->dev.rank && c->peer_base[r]) cudaIpcCloseMemHandle(c->peer_base[r]);
    if (c->segment) cudaFree(c->segment);
    (void)cudaGetLastError();
    delete c;
    return DISTEGNN_OK;
}

extern "C" int distegnn_allreduce_packed(void* comm, float* buf, int64_t count, void* stream) {
    DEGNN_CHECK_ARG(comm, "null comm");
    CommHost* c = (CommHost*)comm;
    DEGNN_CHECK_ARG(c->connected, "comm not connected (distegnn_comm_connect)");
    if (count == 0) return DISTEGNN_OK;
    DEGNN_CHECK_ARG(buf && count > 0, "bad buffer");
    const int64_t slots = (count + c->dev.stride - 1) / c->dev.stride;
    DEGNN_CHECK_ARG(slots <= c->dev.max_slots, "count exceeds the capacity given to distegnn_comm_init");
    allreduce_packed_kernel<<<(unsigned)slots, 256, 0, (cudaStream_t)stream>>>(c->dev, buf, count);
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}
