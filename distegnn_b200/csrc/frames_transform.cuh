// Rigid transforms of the frame assembly's evaluation splits (csrc/frames.cu, DESIGN §23): one rotation R and one
// translation t per (seed, sample), a pure function of those two values, so every rank and every launch that needs a
// sample's transform regenerates the same bits and nothing is stored between launches.
//
//   (o0,o1,o2,o3) = Philox4x32-10(counter = (0, q, i, 0), key = (lo32(s), hi32(s)))
//       q = 2 rotation, 3 translation (the noise of frames_noise.cuh uses q ∈ {0, 1}), i sample index, s seed
//   u_k as in frames_noise.cuh;  z = (r01·cospi(2u1), r01·sinpi(2u1), r23·cospi(2u3), r23·sinpi(2u3)),
//       r01 = sqrt(−2 ln u0), r23 = sqrt(−2 ln u2): four standard normals per counter
//   rotation: the unit quaternion (w, x, y, z) = z(q = 2)/|z(q = 2)| (Haar-uniform on SO(3), det +1), R by the fixed
//       expression of frames_rigid in round-to-nearest fp32; |z|² < 2^-100 (both radii 0) gives R = I.  rotate = 0: R = I
//   translation: t = fp32(translate · (z0, z1, z2)) of q = 3
//
// A position becomes ((R_a0·x0 + R_a1·x1) + R_a2·x2) + t_a and a velocity the same without t, every operation
// round-to-nearest, no contraction.  The production kernels and the testing hook (csrc/testing/frames_transform.cu)
// compile this one definition and produce the same bits.
#pragma once
#include "frames_noise.cuh"

namespace degnn {

enum { XFORM_ROT = 2, XFORM_TRANS = 3 };

// The transform of one assembly launch.  sample_ids [n_samples] (device) is each batch sample's index in the loader's
// sample list; an id outside [0, 2^32) gives NaN in R and t, so every transformed value of that sample is NaN.
struct FramesTransform {
    const int64_t* sample_ids;
    uint64_t seed;
    float translate;
    int rotate;
};

struct Rigid {
    float r[9];   // row-major R
    float t[3];
};

// The four Box–Muller normals of one counter's words (frames_noise.cuh's uniforms and radii, both angles' sin and cos).
__device__ __forceinline__ void transform_normals(uint4 o, float z[4]) {
    const float r01 = sqrtf(-2.f * logf(noise_uniform(o.x)));
    const float r23 = sqrtf(-2.f * logf(noise_uniform(o.z)));
    float s1, c1, s3, c3;
    sincospif(2.f * noise_uniform(o.y), &s1, &c1);
    sincospif(2.f * noise_uniform(o.w), &s3, &c3);
    z[0] = __fmul_rn(r01, c1);
    z[1] = __fmul_rn(r01, s1);
    z[2] = __fmul_rn(r23, c3);
    z[3] = __fmul_rn(r23, s3);
}

// R and t of sample `sample` under `seed`.  R = I + s·(…) with s = 2/|q|², the unit quaternion's matrix without
// normalising q first.
__device__ __forceinline__ void rigid_of(uint64_t seed, uint32_t sample, bool rotate, float translate, Rigid& T) {
    float q[4];
    if (rotate) {
        transform_normals(noise_raw(seed, 0, sample, 0, XFORM_ROT), q);
    } else {
        q[0] = 1.f; q[1] = q[2] = q[3] = 0.f;
    }
    const float w = q[0], x = q[1], y = q[2], z = q[3];
    const float n2 = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(w, w), __fmul_rn(x, x)), __fmul_rn(y, y)), __fmul_rn(z, z));
    if (!rotate || n2 < 0x1p-100f) {
        T.r[0] = 1.f; T.r[1] = 0.f; T.r[2] = 0.f;
        T.r[3] = 0.f; T.r[4] = 1.f; T.r[5] = 0.f;
        T.r[6] = 0.f; T.r[7] = 0.f; T.r[8] = 1.f;
    } else {
        const float s = __fdiv_rn(2.f, n2);
        const float xx = __fmul_rn(x, x), yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
        const float xy = __fmul_rn(x, y), xz = __fmul_rn(x, z), yz = __fmul_rn(y, z);
        const float wx = __fmul_rn(w, x), wy = __fmul_rn(w, y), wz = __fmul_rn(w, z);
        T.r[0] = __fsub_rn(1.f, __fmul_rn(s, __fadd_rn(yy, zz)));
        T.r[1] = __fmul_rn(s, __fsub_rn(xy, wz));
        T.r[2] = __fmul_rn(s, __fadd_rn(xz, wy));
        T.r[3] = __fmul_rn(s, __fadd_rn(xy, wz));
        T.r[4] = __fsub_rn(1.f, __fmul_rn(s, __fadd_rn(xx, zz)));
        T.r[5] = __fmul_rn(s, __fsub_rn(yz, wx));
        T.r[6] = __fmul_rn(s, __fsub_rn(xz, wy));
        T.r[7] = __fmul_rn(s, __fadd_rn(yz, wx));
        T.r[8] = __fsub_rn(1.f, __fmul_rn(s, __fadd_rn(xx, yy)));
    }
    float zt[4];
    transform_normals(noise_raw(seed, 0, sample, 0, XFORM_TRANS), zt);
#pragma unroll
    for (int d = 0; d < 3; ++d) T.t[d] = __fmul_rn(translate, zt[d]);
}

// The transform of batch sample b.
__device__ __forceinline__ void frames_rigid(const FramesTransform& xf, int b, Rigid& T) {
    const int64_t id = __ldg(xf.sample_ids + b);
    rigid_of(xf.seed, (uint32_t)id, xf.rotate != 0, xf.translate, T);
    if (id < 0 || id > (int64_t)UINT32_MAX) {
        const float nan = __int_as_float(0x7fc00000);
#pragma unroll
        for (int k = 0; k < 9; ++k) T.r[k] = nan;
        T.t[0] = T.t[1] = T.t[2] = nan;
    }
}

// v ← R·v (+ t for a position), in the fixed order ((R_a0·v0 + R_a1·v1) + R_a2·v2) + t_a.
__device__ __forceinline__ void rigid_apply(const Rigid& T, float v[3], bool position) {
    float o[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        o[a] = __fadd_rn(__fadd_rn(__fmul_rn(T.r[a * 3], v[0]), __fmul_rn(T.r[a * 3 + 1], v[1])),
                         __fmul_rn(T.r[a * 3 + 2], v[2]));
        if (position) o[a] = __fadd_rn(o[a], T.t[a]);
    }
    v[0] = o[0]; v[1] = o[1]; v[2] = o[2];
}

}  // namespace degnn
