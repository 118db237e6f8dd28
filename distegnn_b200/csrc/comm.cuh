// Device side of the virtual-node sync: a one-shot, push-based SUM all-reduce of small packed buffers over NVLink peer
// memory (replaces weighted_average_reduce / _AllReduce, models/FastEGNN.py:10-43, 310-319).
//
// Every rank owns one "segment" of device memory that all peers map (CUDA IPC).  A call reduces `count` floats cut into
// SLOTS of at most `stride` floats; slot s is handled by exactly one CTA on every rank:
//   1. push   : the CTA stores its slot's values into data[parity][my_rank][s] of EVERY rank's segment (its own included)
//   2. signal : after a system-scope fence, flag[parity][my_rank][s] of every rank's segment := epoch
//   3. wait   : until the local flags of all ranks for this slot carry the epoch (bounded spin; a timeout sets `status`)
//   4. reduce : Σ_r data[parity][r][s] in RANK ORDER — every rank adds the same numbers in the same order, so the result is
//               bit-identical on all ranks (the reference relies on NCCL for that property, FastEGNN.py:29-31)
// The epoch of a slot lives in the segment and is advanced by the kernel itself, so the same launch can be replayed from a
// CUDA graph.  parity = epoch & 1 double-buffers the data: a rank can only be one call ahead of its slowest peer (it needs
// the peer's flag of call e+1, which the peer sends after it finished reading call e), so two buffers are enough.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace degnn {

constexpr int COMM_MAX_WORLD = 16;

struct CommDev {
    int rank, world;
    int max_slots;            // slots per call
    int stride;               // floats per slot
    float* data[COMM_MAX_WORLD];       // per rank: [2][world][max_slots][stride]
    unsigned* flags[COMM_MAX_WORLD];   // per rank: [2][world][max_slots]
    unsigned* epoch;          // local: [max_slots]
    unsigned* status;         // local: [0] != 0 after a timeout
    unsigned long long timeout_ns;
};

__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(unsigned* p, unsigned v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ float ld_volatile_f32(const float* p) {
    float v;
    asm volatile("ld.volatile.global.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

// The default pause of comm_slot_allreduce: none.
struct NoPause {
    __device__ __forceinline__ void operator()() const {}
};

// All-reduce (SUM) of slot `slot`: `vals[0:n]` (global or shared memory of this CTA, n <= stride) in place.  Must be called
// by ALL threads of the CTA; returns after a __syncthreads(), with vals holding the sum over the ranks.  `pause()` is called
// by every thread between the wait and the reduce: the window in which a faster peer may already push the next call (the
// parity double buffer keeps it out of the data being reduced).  Tests use it to make the ranks drift; the product passes
// none.
template <class Pause = NoPause>
__device__ __forceinline__ void comm_slot_allreduce(const CommDev& cd, int slot, float* vals, int n, Pause pause = {}) {
    __shared__ unsigned s_epoch;
    const int tid = threadIdx.x, nt = blockDim.x;
    if (tid == 0) s_epoch = cd.epoch[slot] + 1u;
    __syncthreads();
    const unsigned e = s_epoch;
    const size_t par = e & 1u;
    const size_t per_rank = (size_t)cd.max_slots * cd.stride;
    const size_t mine = (par * cd.world + cd.rank) * per_rank + (size_t)slot * cd.stride;
    // 1. push
    for (int i = tid; i < n; i += nt) {
        const float v = vals[i];
        for (int r = 0; r < cd.world; ++r) cd.data[r][mine + i] = v;
    }
    __syncthreads();
    // 2. signal (one thread per destination rank)
    if (tid < cd.world) {
        __threadfence_system();
        st_release_sys(cd.flags[tid] + (par * cd.world + cd.rank) * cd.max_slots + slot, e);
    }
    // 3. wait (one thread per source rank)
    if (tid < cd.world) {
        const unsigned* f = cd.flags[cd.rank] + (par * cd.world + tid) * cd.max_slots + slot;
        const unsigned long long t0 = globaltimer_ns();
        unsigned spins = 0;
        while ((int)(ld_acquire_sys(f) - e) < 0) {
            if ((++spins & 1023u) == 0 && globaltimer_ns() - t0 > cd.timeout_ns) {
                atomicExch(cd.status, 1u);
                break;
            }
        }
    }
    __syncthreads();
    pause();
    // 4. reduce in rank order
    const float* base = cd.data[cd.rank] + par * cd.world * per_rank + (size_t)slot * cd.stride;
    for (int i = tid; i < n; i += nt) {
        float s = ld_volatile_f32(base + i);
        for (int r = 1; r < cd.world; ++r) s += ld_volatile_f32(base + (size_t)r * per_rank + i);
        vals[i] = s;
    }
    if (tid == 0) cd.epoch[slot] = e;
    __syncthreads();
}

// Layout of one rank's segment: flags [2][world][max_slots], epoch [max_slots], status, data [2][world][max_slots][stride].
struct SegLayout {
    size_t flags_off, epoch_off, status_off, data_off, total;
};
inline size_t seg_align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
inline SegLayout seg_layout(int world, int max_slots, int stride) {
    SegLayout s;
    s.flags_off = 0;
    s.epoch_off = seg_align_up(s.flags_off + sizeof(unsigned) * 2 * (size_t)world * max_slots, 256);
    s.status_off = seg_align_up(s.epoch_off + sizeof(unsigned) * (size_t)max_slots, 256);
    s.data_off = seg_align_up(s.status_off + 64, 256);
    s.total = seg_align_up(s.data_off + sizeof(float) * 2 * (size_t)world * max_slots * stride, 256);
    return s;
}

// host handle behind the opaque `void* comm` of the C ABI
struct CommHost {
    CommDev dev;
    void* segment;             // local segment (cudaMalloc)
    size_t segment_bytes;
    void* peer_base[COMM_MAX_WORLD];
    bool connected;
    int device;
};

}  // namespace degnn
