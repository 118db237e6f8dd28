// Frame assembly: the per-sample arithmetic of the reference's data pipeline on the device (distegnn_b200/frames.py).
//
// The reference builds every training sample once on the host (datasets/process_dataset.py:61-115 N-body, :239-277 and
// :334-347 Water-3D, :480-557 Fluid113K) and caches it.  Here the loader stages the raw frames a batch needs and
//   distegnn_frames_assemble   per scene: loc_mean (fp64 sums over the WHOLE frame, fixed order) and the max of the
//                              normalised static column, both before any split (distribute_graphs.py:32, :346 then :348);
//                              per node of this rank: the gathers, v, ‖v‖ and the normalised column, data_batch
// builds this rank's node arrays in two launches, without allocating or synchronising (capturable).  With a horizon K > 1
//   distegnn_frames_targets    gathers the staged frames pos[f + 2Δ] .. pos[f + KΔ] into targets[1:] the same way
// (one more launch; targets[0] is the assembly's target).
//   distegnn_frames_assemble_noise   the same launches with training noise (frames_noise.cuh, DESIGN §22): ε_x is added
//                              to x (also inside the whole-scene sum of loc_mean) and to every target row, ε_v to v
//                              before ‖v‖; the kernels regenerate a node's ε wherever they need it
//   distegnn_frames_assemble_transform   the same launches with a rigid transform per sample (frames_transform.cuh,
//                              DESIGN §23): every staged position becomes R·x + t and every staged velocity R·v as it
//                              is gathered, before any of the recipe's arithmetic
#include "common.cuh"
#include "frames_noise.cuh"
#include "frames_transform.cuh"

namespace degnn {

constexpr int RED_THREADS = 512;

struct FramesArgs {
    int recipe, B, S;
    int64_t n_frame, n_out;
    const float* x0;            // [n_frame,3] pos[f]
    const float* x1;            // [n_frame,3] pos[f+1] (Water-3D) or vel[f]
    const float* xt;            // [n_frame,3] pos[f+Δ]
    const float* stat;          // [n_frame,S]
    const int64_t* scene_ptr;   // [B+1]
    const int64_t* out_ptr;     // [B+1]
    const int32_t* index;       // [n_out] or null
    float *feat, *loc, *vel, *attr, *target;
    int64_t* batch;
    float *loc_mean, *scene_max;
};

// One block per scene: Σx in fp64 by a fixed per-thread stride and a fixed tree, so the result does not depend on
// scheduling; the max of static column 0 (order-independent).  NOISE: Σ(x + ε_x) over every node of the scene.  XFORM:
// Σ(R·x + t) over every node of the scene.
template <bool NOISE, bool XFORM>
__global__ void __launch_bounds__(RED_THREADS) frames_scene_kernel(const FramesArgs a, const FramesNoise nz,
                                                                    const FramesTransform xf) {
    __shared__ double ssum[3][RED_THREADS];
    __shared__ float smax[RED_THREADS];
    const int b = blockIdx.x, t = threadIdx.x;
    const int64_t lo = a.scene_ptr[b], hi = a.scene_ptr[b + 1];
    double s0 = 0.0, s1 = 0.0, s2 = 0.0;
    float m = -INFINITY;
    Rigid T;
    if (XFORM) frames_rigid(xf, b, T);
    for (int64_t i = lo + t; i < hi; i += RED_THREADS) {
        float x[3] = {__ldg(a.x0 + i * 3), __ldg(a.x0 + i * 3 + 1), __ldg(a.x0 + i * 3 + 2)};
        if (XFORM) rigid_apply(T, x, true);
        if (NOISE) {
            float e[3];
            frames_noise(nz, b, i - lo, NOISE_POS, e);
#pragma unroll
            for (int d = 0; d < 3; ++d) x[d] = __fadd_rn(x[d], e[d]);
        }
        s0 += (double)x[0];
        s1 += (double)x[1];
        s2 += (double)x[2];
        m = fmaxf(m, __ldg(a.stat + i * a.S));
    }
    ssum[0][t] = s0; ssum[1][t] = s1; ssum[2][t] = s2; smax[t] = m;
    __syncthreads();
    for (int w = RED_THREADS / 2; w > 0; w >>= 1) {
        if (t < w) {
#pragma unroll
            for (int d = 0; d < 3; ++d) ssum[d][t] += ssum[d][t + w];
            smax[t] = fmaxf(smax[t], smax[t + w]);
        }
        __syncthreads();
    }
    if (t == 0) {
        const double n = (double)(hi - lo);
#pragma unroll
        for (int d = 0; d < 3; ++d) a.loc_mean[b * 3 + d] = __double2float_rn(ssum[d][0] / n);
        a.scene_max[b] = smax[0];
    }
}

__device__ __forceinline__ int sample_of(const int64_t* ptr, int B, int64_t k) {
    int lo = 0, hi = B - 1;                    // last b with ptr[b] <= k
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(ptr + mid) <= k) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// ‖v‖ = sqrt((vx·vx + vy·vy) + vz·vz), every operation round-to-nearest, no contraction (the reference's order).
__device__ __forceinline__ float speed_of(const float v[3]) {
    return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(v[0], v[0]), __fmul_rn(v[1], v[1])), __fmul_rn(v[2], v[2])));
}

// One thread per output node.  Gathers are copies; v, ‖v‖ and the division are round-to-nearest fp32 operations in the
// reference's order (no contraction).  NOISE: x, v and the target get one fp32 add of ε_x, ε_v, ε_x (v first computed as
// without noise), and ‖v‖ is taken of the noisy v.  XFORM: x, the target and pos[f+1] (Water-3D) become R·x + t and
// vel[f] becomes R·v as they are gathered; v, ‖v‖ and the rest follow from those as without the transform.
template <bool NOISE, bool XFORM>
__global__ void __launch_bounds__(256) frames_node_kernel(const FramesArgs a, const FramesNoise nz,
                                                          const FramesTransform xf) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < a.n_out; k += (int64_t)gridDim.x * blockDim.x) {
        const int b = sample_of(a.out_ptr, a.B, k);
        const int64_t base = __ldg(a.scene_ptr + b), n = __ldg(a.scene_ptr + b + 1) - base;
        const int64_t li = a.index ? (int64_t)__ldg(a.index + k) : k - __ldg(a.out_ptr + b);
        const bool ok = li >= 0 && li < n;     // the host validates the index lists; never read outside the scene
        const int64_t g = base + (ok ? li : 0);
        const float nan = __int_as_float(0x7fc00000);
        float x[3], v[3], y[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            x[d] = ok ? __ldg(a.x0 + g * 3 + d) : nan;
            y[d] = ok ? __ldg(a.xt + g * 3 + d) : nan;
            const float w = ok ? __ldg(a.x1 + g * 3 + d) : nan;
            v[d] = (XFORM || a.recipe != DISTEGNN_FRAMES_WATER3D) ? w : __fsub_rn(w, x[d]);
        }
        if (XFORM) {
            Rigid T;
            frames_rigid(xf, b, T);
            const bool w3d = a.recipe == DISTEGNN_FRAMES_WATER3D;      // v holds pos[f+1] (a position) or vel[f]
            rigid_apply(T, x, true);
            rigid_apply(T, y, true);
            rigid_apply(T, v, w3d);
            if (w3d) {
#pragma unroll
                for (int d = 0; d < 3; ++d) v[d] = __fsub_rn(v[d], x[d]);
            }
        }
        if (NOISE) {
            float ex[3], ev[3];
            frames_noise(nz, b, li, NOISE_POS, ex);
            frames_noise(nz, b, li, NOISE_VEL, ev);
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                x[d] = __fadd_rn(x[d], ex[d]);
                y[d] = __fadd_rn(y[d], ex[d]);
                v[d] = __fadd_rn(v[d], ev[d]);
            }
        }
        const float speed = speed_of(v);
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            a.loc[k * 3 + d] = x[d];
            a.vel[k * 3 + d] = v[d];
            a.target[k * 3 + d] = y[d];
        }
        if (a.recipe == DISTEGNN_FRAMES_LARGEFLUID) {         // [viscosity, mass, ‖v‖] / [viscosity, mass]
            const float s0 = ok ? __ldg(a.stat + g * 2) : nan, s1 = ok ? __ldg(a.stat + g * 2 + 1) : nan;
            a.feat[k * 3] = s0; a.feat[k * 3 + 1] = s1; a.feat[k * 3 + 2] = speed;
            a.attr[k * 2] = s0; a.attr[k * 2 + 1] = s1;
        } else {                                              // [‖v‖, s / max(s)] / [s]
            const float s = ok ? __ldg(a.stat + g) : nan;
            a.feat[k * 2] = speed;
            a.feat[k * 2 + 1] = __fdiv_rn(s, __ldg(a.scene_max + b));
            a.attr[k] = s;
        }
        a.batch[k] = b;
    }
}

// One thread per (horizon step t >= 1, output node): targets[t] = frame 2 + t of the staged block (pos[f + (t+1)Δ]),
// by the node kernel's scene offsets and index.  Copies only; NOISE: every row plus the node's ε_x (one fp32 add);
// XFORM: every row R·x + t.
template <bool NOISE, bool XFORM>
__global__ void __launch_bounds__(256) frames_targets_kernel(int B, int64_t n_frame, int64_t n_out, int K,
                                                             const float* frames, const int64_t* scene_ptr,
                                                             const int64_t* out_ptr, const int32_t* index,
                                                             float* targets, const FramesNoise nz,
                                                             const FramesTransform xf) {
    const int64_t total = (int64_t)(K - 1) * n_out;
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += (int64_t)gridDim.x * blockDim.x) {
        const int64_t t = q / n_out + 1, k = q - (t - 1) * n_out;
        const int b = sample_of(out_ptr, B, k);
        const int64_t base = __ldg(scene_ptr + b), n = __ldg(scene_ptr + b + 1) - base;
        const int64_t li = index ? (int64_t)__ldg(index + k) : k - __ldg(out_ptr + b);
        const bool ok = li >= 0 && li < n;
        const float* src = frames + ((2 + t) * n_frame + base + (ok ? li : 0)) * 3;
        float* dst = targets + (t * n_out + k) * 3;
        const float nan = __int_as_float(0x7fc00000);
        if (NOISE) {
            float e[3];
            frames_noise(nz, b, li, NOISE_POS, e);
#pragma unroll
            for (int d = 0; d < 3; ++d) dst[d] = __fadd_rn(ok ? __ldg(src + d) : nan, e[d]);
        } else if (XFORM) {
            Rigid T;
            frames_rigid(xf, b, T);
            float x[3] = {ok ? __ldg(src) : nan, ok ? __ldg(src + 1) : nan, ok ? __ldg(src + 2) : nan};
            rigid_apply(T, x, true);
#pragma unroll
            for (int d = 0; d < 3; ++d) dst[d] = x[d];
        } else {
#pragma unroll
            for (int d = 0; d < 3; ++d) dst[d] = ok ? __ldg(src + d) : nan;
        }
    }
}

static unsigned node_grid(int64_t n) {
    const int64_t cap = 8 * (int64_t)sm_count();
    const int64_t g = (n + 255) / 256;
    return (unsigned)(g < 1 ? 1 : (g > cap ? cap : g));
}

// The assembly's argument checks and kernel arguments, shared by both assembly entry points (errors name `who`).
static int frames_args(const char* who, int recipe, int n_samples, int64_t n_frame_nodes, int64_t n_out,
                       const float* frames, const float* statics, const int64_t* scene_ptr, const int64_t* out_ptr,
                       const int32_t* index, float* node_feat, float* node_loc, float* node_vel, float* node_attr,
                       float* target, int64_t* data_batch, float* loc_mean, float* scene_max, FramesArgs& a) {
    const char* bad = nullptr;
    if (!(recipe == DISTEGNN_FRAMES_NBODY || recipe == DISTEGNN_FRAMES_WATER3D || recipe == DISTEGNN_FRAMES_LARGEFLUID))
        bad = "unknown recipe";
    else if (!(n_samples >= 1 && n_frame_nodes >= 0 && n_out >= 0))
        bad = "bad size";
    else if (!(index || n_out == n_frame_nodes))
        bad = "without an index list every node is assembled (n_out == n_frame_nodes)";
    else if (!(scene_ptr && out_ptr && loc_mean && scene_max) || !(n_frame_nodes == 0 || (frames && statics)) ||
             !(n_out == 0 || (node_feat && node_loc && node_vel && node_attr && target && data_batch)))
        bad = "null pointer";
    if (bad) {
        set_error("%s: %s", who, bad);
        return DISTEGNN_EINVAL;
    }
    a.recipe = recipe; a.B = n_samples; a.S = recipe == DISTEGNN_FRAMES_LARGEFLUID ? 2 : 1;
    a.n_frame = n_frame_nodes; a.n_out = n_out;
    a.x0 = frames; a.x1 = frames + n_frame_nodes * 3; a.xt = frames + n_frame_nodes * 6; a.stat = statics;
    a.scene_ptr = scene_ptr; a.out_ptr = out_ptr; a.index = index;
    a.feat = node_feat; a.loc = node_loc; a.vel = node_vel; a.attr = node_attr; a.target = target; a.batch = data_batch;
    a.loc_mean = loc_mean; a.scene_max = scene_max;
    return DISTEGNN_OK;
}

}  // namespace degnn

extern "C" int distegnn_frames_assemble(int recipe, int n_samples, int64_t n_frame_nodes, int64_t n_out,
                                        const float* frames, const float* statics, const int64_t* scene_ptr,
                                        const int64_t* out_ptr, const int32_t* index, float* node_feat, float* node_loc,
                                        float* node_vel, float* node_attr, float* target, int64_t* data_batch,
                                        float* loc_mean, float* scene_max, void* stream) {
    using namespace degnn;
    FramesArgs a;
    const int rc = frames_args(__func__, recipe, n_samples, n_frame_nodes, n_out, frames, statics, scene_ptr, out_ptr,
                               index, node_feat, node_loc, node_vel, node_attr, target, data_batch, loc_mean, scene_max,
                               a);
    if (rc != DISTEGNN_OK) return rc;
    const FramesNoise none{};
    frames_scene_kernel<false, false><<<n_samples, RED_THREADS, 0, (cudaStream_t)stream>>>(a, none, FramesTransform{});
    DEGNN_CHECK_LAUNCH();
    if (n_out > 0) {
        frames_node_kernel<false, false><<<node_grid(n_out), 256, 0, (cudaStream_t)stream>>>(a, none, FramesTransform{});
        DEGNN_CHECK_LAUNCH();
    }
    return DISTEGNN_OK;
}

extern "C" int distegnn_frames_targets(int n_samples, int64_t n_frame_nodes, int64_t n_out, int horizon,
                                       const float* frames, const int64_t* scene_ptr, const int64_t* out_ptr,
                                       const int32_t* index, float* targets, void* stream) {
    using namespace degnn;
    DEGNN_CHECK_ARG(n_samples >= 1 && n_frame_nodes >= 0 && n_out >= 0 && horizon >= 1, "bad size");
    DEGNN_CHECK_ARG(index || n_out == n_frame_nodes, "without an index list every node is gathered (n_out == n_frame_nodes)");
    if (horizon == 1 || n_out == 0) return DISTEGNN_OK;
    DEGNN_CHECK_ARG(frames && scene_ptr && out_ptr && targets, "null pointer");
    frames_targets_kernel<false, false><<<node_grid((int64_t)(horizon - 1) * n_out), 256, 0, (cudaStream_t)stream>>>(
        n_samples, n_frame_nodes, n_out, horizon, frames, scene_ptr, out_ptr, index, targets, FramesNoise{},
        FramesTransform{});
    DEGNN_CHECK_LAUNCH();
    return DISTEGNN_OK;
}

extern "C" int distegnn_frames_assemble_noise(int recipe, int n_samples, int64_t n_frame_nodes, int64_t n_out,
                                              int horizon, const float* frames, const float* statics,
                                              const int64_t* scene_ptr, const int64_t* out_ptr, const int32_t* index,
                                              float* node_feat, float* node_loc, float* node_vel, float* node_attr,
                                              float* targets, int64_t* data_batch, float* loc_mean, float* scene_max,
                                              const int64_t* sample_ids, uint64_t seed, uint32_t epoch, float sigma_x,
                                              float sigma_v, void* stream) {
    using namespace degnn;
    DEGNN_CHECK_ARG(horizon >= 1, "horizon must be >= 1");
    DEGNN_CHECK_ARG(isfinite(sigma_x) && isfinite(sigma_v) && sigma_x >= 0.f && sigma_v >= 0.f,
                    "sigma_x and sigma_v must be finite and >= 0");
    DEGNN_CHECK_ARG(sample_ids, "null sample_ids");
    FramesArgs a;
    const int rc = frames_args(__func__, recipe, n_samples, n_frame_nodes, n_out, frames, statics, scene_ptr, out_ptr,
                               index, node_feat, node_loc, node_vel, node_attr, targets, data_batch, loc_mean, scene_max,
                               a);
    if (rc != DISTEGNN_OK) return rc;
    const FramesNoise nz{sample_ids, seed, epoch, sigma_x, sigma_v};
    const FramesTransform none{};
    frames_scene_kernel<true, false><<<n_samples, RED_THREADS, 0, (cudaStream_t)stream>>>(a, nz, none);
    DEGNN_CHECK_LAUNCH();
    if (n_out > 0) {
        frames_node_kernel<true, false><<<node_grid(n_out), 256, 0, (cudaStream_t)stream>>>(a, nz, none);
        DEGNN_CHECK_LAUNCH();
        if (horizon > 1) {
            frames_targets_kernel<true, false><<<node_grid((int64_t)(horizon - 1) * n_out), 256, 0,
                                                 (cudaStream_t)stream>>>(
                n_samples, n_frame_nodes, n_out, horizon, frames, scene_ptr, out_ptr, index, targets, nz, none);
            DEGNN_CHECK_LAUNCH();
        }
    }
    return DISTEGNN_OK;
}

extern "C" int distegnn_frames_assemble_transform(int recipe, int n_samples, int64_t n_frame_nodes, int64_t n_out,
                                                  int horizon, const float* frames, const float* statics,
                                                  const int64_t* scene_ptr, const int64_t* out_ptr,
                                                  const int32_t* index, float* node_feat, float* node_loc,
                                                  float* node_vel, float* node_attr, float* targets,
                                                  int64_t* data_batch, float* loc_mean, float* scene_max,
                                                  const int64_t* sample_ids, uint64_t seed, int rotate,
                                                  float translate, void* stream) {
    using namespace degnn;
    DEGNN_CHECK_ARG(horizon >= 1, "horizon must be >= 1");
    DEGNN_CHECK_ARG(rotate == 0 || rotate == 1, "rotate must be 0 or 1");
    DEGNN_CHECK_ARG(isfinite(translate) && translate >= 0.f, "translate must be finite and >= 0");
    DEGNN_CHECK_ARG(sample_ids, "null sample_ids");
    FramesArgs a;
    const int rc = frames_args(__func__, recipe, n_samples, n_frame_nodes, n_out, frames, statics, scene_ptr, out_ptr,
                               index, node_feat, node_loc, node_vel, node_attr, targets, data_batch, loc_mean, scene_max,
                               a);
    if (rc != DISTEGNN_OK) return rc;
    const FramesNoise none{};
    const FramesTransform xf{sample_ids, seed, translate, rotate};
    frames_scene_kernel<false, true><<<n_samples, RED_THREADS, 0, (cudaStream_t)stream>>>(a, none, xf);
    DEGNN_CHECK_LAUNCH();
    if (n_out > 0) {
        frames_node_kernel<false, true><<<node_grid(n_out), 256, 0, (cudaStream_t)stream>>>(a, none, xf);
        DEGNN_CHECK_LAUNCH();
        if (horizon > 1) {
            frames_targets_kernel<false, true><<<node_grid((int64_t)(horizon - 1) * n_out), 256, 0,
                                                 (cudaStream_t)stream>>>(
                n_samples, n_frame_nodes, n_out, horizon, frames, scene_ptr, out_ptr, index, targets, none, xf);
            DEGNN_CHECK_LAUNCH();
        }
    }
    return DISTEGNN_OK;
}
