// N-body dataset generation: the reference's charged-particle simulator (dataset_generation/nbody/system.py,
// physical_objects.py) in fp64 on the device: isolated bodies, and sticks and hinges (DESIGN §25).
//
// Per step and body i, in this order and with no FMA contraction (every product and sum rounds on its own):
//   ‖x‖² = (x·x + y·y) + z·z,  dot = (x_i x_j + y_i y_j) + z_i z_j,  l2 = (‖x_i‖² + ‖x_j‖²) − 2·dot
//   s_ij = (q_i q_j) / (l2·sqrt(l2)),  F_i = Σ_{j = 0..n−1} s_ij·(x_i − x_j)  summed in ascending j, the j = i term +0.0
//   F clamped to ±max_f per component (NaN passes),  v ← v + F·dt,  x ← x + v·dt
// A step fails the reference's check when some off-diagonal |s_ij| is not > 1e-10 (NaN included); status[s] keeps the
// first failing step of system s (−1: none so far).  Step t is recorded when t % sample_freq == 0, after it runs.
//
// Two paths, picked by the number of bodies; both give the same bits:
//   n <= 1024  nbody_cta_kernel: one thread per body, max(1, 512 / n) whole systems per CTA (so that small systems
//              fill the warps) in shared memory; one launch runs the steps up to the next recorded one and writes that
//              frame
//   n >  1024  nbody_force_tiled_kernel then nbody_drift_kernel per step: each thread owns body i and walks the bodies
//              j in shared-memory tiles, in ascending order; the force kernel updates v (only its owner reads v_i),
//              the drift kernel x, so no CTA reads a position another CTA has already moved
// Sticks and hinges (distegnn_nbody_simulate_objects) take the same clamped force; then isolated bodies kick and drift
// as above and each object restates Stick.update / Hinge.update on its own bodies (see "Sticks and hinges" below).
#include <climits>

#include "common.cuh"

namespace degnn {

constexpr int NBODY_CTA_MAX = 1024;
constexpr int NBODY_CTA_PACK = 512;     // bodies of several small systems per CTA
constexpr int NBODY_TILE = 256;

struct NbodyArgs {
    int S, n;
    int64_t R;                  // frames recorded by this call (the frames buffers are [S, R, n, 3])
    double dt, max_f;
    double *x, *v;              // [S, n, 3], read and written in place
    const double* q;            // [S, n]
    double *fx, *fv;            // [S, R, n, 3]
    int64_t* status;            // [S]
};

__device__ __forceinline__ double norm2(double x, double y, double z) {
    return __dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z));
}

// One term of F_i in place: body j at (xj, yj, zj), ‖x_j‖² nj, charge qj.  Sets bad when j != i and |s_ij| is not
// above 1e-10.
__device__ __forceinline__ void pair_term(const double xi, const double yi, const double zi, const double ni,
                                          const double qi, const double xj, const double yj, const double zj,
                                          const double nj, const double qj, const bool self, double& f0, double& f1,
                                          double& f2, bool& bad) {
    const double dot = __dadd_rn(__dadd_rn(__dmul_rn(xi, xj), __dmul_rn(yi, yj)), __dmul_rn(zi, zj));
    const double l2 = __dsub_rn(__dadd_rn(ni, nj), __dmul_rn(2.0, dot));
    const double s = __ddiv_rn(__dmul_rn(qi, qj), __dmul_rn(l2, __dsqrt_rn(l2)));
    bad |= !self && !(fabs(s) > 1e-10);
    f0 = __dadd_rn(f0, self ? 0.0 : __dmul_rn(s, __dsub_rn(xi, xj)));
    f1 = __dadd_rn(f1, self ? 0.0 : __dmul_rn(s, __dsub_rn(yi, yj)));
    f2 = __dadd_rn(f2, self ? 0.0 : __dmul_rn(s, __dsub_rn(zi, zj)));
}

__device__ __forceinline__ double clamp_f(double f, double m) {
    if (f > m) return m;
    if (f < -m) return -m;
    return f;                   // NaN passes, as numpy's masked assignment leaves it
}

__device__ __forceinline__ void kick(double& v, double f, double m, double dt) { v = __dadd_rn(v, __dmul_rn(clamp_f(f, m), dt)); }

// Systems blockIdx.x·per_cta .. (at most per_cta of them, contiguous in memory), thread k on body k of them: steps
// t0 .. t0 + steps − 1, then (slot >= 0) the state into frame slot.  Shared memory: (x, y), (z, ‖x‖²) and q of every
// body of the CTA.
__global__ void __launch_bounds__(NBODY_CTA_MAX) nbody_cta_kernel(const NbodyArgs a, const int per_cta,
                                                                  const int64_t t0, const int steps,
                                                                  const int64_t slot) {
    extern __shared__ double2 sm[];
    const int n = a.n, s0 = blockIdx.x * per_cta, G = min(per_cta, a.S - s0), k = threadIdx.x;
    double2* sxy = sm;
    double2* szn = sm + per_cta * n;
    double* sq = reinterpret_cast<double*>(sm + 2 * per_cta * n);
    __shared__ unsigned long long first_bad[NBODY_CTA_PACK / 2];
    const bool own = k < G * n;
    const int g = k / n, i = k - g * n, s = s0 + g;
    const double2* gxy = sxy + g * n;       // this thread's system in shared memory
    const double2* gzn = szn + g * n;
    const double* gq = sq + g * n;
    const int64_t row = ((int64_t)s0 * n + k) * 3;
    double x0 = 0.0, x1 = 0.0, x2 = 0.0, v0 = 0.0, v1 = 0.0, v2 = 0.0, qi = 0.0;
    if (own) {
        x0 = a.x[row], x1 = a.x[row + 1], x2 = a.x[row + 2];
        v0 = a.v[row], v1 = a.v[row + 1], v2 = a.v[row + 2];
        qi = a.q[(int64_t)s0 * n + k];
        sq[k] = qi;
    }
    if (k < per_cta) first_bad[k] = ULLONG_MAX;
    unsigned long long my_bad = ULLONG_MAX;
    for (int u = 0; u < steps; ++u) {
        double ni = 0.0;
        if (own) {
            ni = norm2(x0, x1, x2);
            sxy[k] = make_double2(x0, x1);
            szn[k] = make_double2(x2, ni);
        }
        __syncthreads();
        if (own) {
            double f0 = 0.0, f1 = 0.0, f2 = 0.0;
            bool bad = false;
            for (int j = 0; j < n; ++j) {
                const double2 xy = gxy[j], zn = gzn[j];
                pair_term(x0, x1, x2, ni, qi, xy.x, xy.y, zn.x, zn.y, gq[j], j == i, f0, f1, f2, bad);
            }
            if (bad && my_bad == ULLONG_MAX) my_bad = (unsigned long long)(t0 + u);
            kick(v0, f0, a.max_f, a.dt);
            kick(v1, f1, a.max_f, a.dt);
            kick(v2, f2, a.max_f, a.dt);
            x0 = __dadd_rn(x0, __dmul_rn(v0, a.dt));
            x1 = __dadd_rn(x1, __dmul_rn(v1, a.dt));
            x2 = __dadd_rn(x2, __dmul_rn(v2, a.dt));
        }
        __syncthreads();        // every read of this step's positions is done before the next step writes them
    }
    if (my_bad != ULLONG_MAX) atomicMin(&first_bad[g], my_bad);
    if (own) {
        a.x[row] = x0, a.x[row + 1] = x1, a.x[row + 2] = x2;
        a.v[row] = v0, a.v[row + 1] = v1, a.v[row + 2] = v2;
        if (slot >= 0) {
            const int64_t f = (((int64_t)s * a.R + slot) * n + i) * 3;
            a.fx[f] = x0, a.fx[f + 1] = x1, a.fx[f + 2] = x2;
            a.fv[f] = v0, a.fv[f + 1] = v1, a.fv[f + 2] = v2;
        }
    }
    __syncthreads();
    if (k < G && first_bad[k] != ULLONG_MAX && a.status[s0 + k] < 0) a.status[s0 + k] = (int64_t)first_bad[k];
}

// F_i of body i (own: i < n) of system s, the bodies j through shared memory a tile at a time; every thread of the
// CTA takes part in the tile loads.
__device__ __forceinline__ void tiled_force(const NbodyArgs& a, const int s, const int i, const bool own, double& f0,
                                            double& f1, double& f2, bool& bad) {
    __shared__ double2 sxy[NBODY_TILE], szn[NBODY_TILE];
    __shared__ double sq[NBODY_TILE];
    const int n = a.n;
    const double* xs = a.x + (int64_t)s * n * 3;
    const double* qs = a.q + (int64_t)s * n;
    double x0 = 0.0, x1 = 0.0, x2 = 0.0, qi = 0.0, ni = 0.0;
    if (own) {
        x0 = xs[i * 3], x1 = xs[i * 3 + 1], x2 = xs[i * 3 + 2];
        qi = qs[i];
        ni = norm2(x0, x1, x2);
    }
    for (int base = 0; base < n; base += NBODY_TILE) {
        const int j = base + threadIdx.x;
        if (j < n) {
            const double y0 = xs[j * 3], y1 = xs[j * 3 + 1], y2 = xs[j * 3 + 2];
            sxy[threadIdx.x] = make_double2(y0, y1);
            szn[threadIdx.x] = make_double2(y2, norm2(y0, y1, y2));
            sq[threadIdx.x] = qs[j];
        }
        __syncthreads();
        if (own) {
            const int m = min(NBODY_TILE, n - base);
            for (int jj = 0; jj < m; ++jj) {
                const double2 xy = sxy[jj], zn = szn[jj];
                pair_term(x0, x1, x2, ni, qi, xy.x, xy.y, zn.x, zn.y, sq[jj], base + jj == i, f0, f1, f2, bad);
            }
        }
        __syncthreads();
    }
}

// Step t, forces and kick: CTA b of system s owns bodies b·TILE ..; the bodies j come through shared memory a tile at
// a time.
__global__ void __launch_bounds__(NBODY_TILE) nbody_force_tiled_kernel(const NbodyArgs a, const int64_t t) {
    const int n = a.n, nb = (n + NBODY_TILE - 1) / NBODY_TILE;
    const int s = blockIdx.x / nb, i = (blockIdx.x % nb) * NBODY_TILE + threadIdx.x;
    const bool own = i < n;
    double f0 = 0.0, f1 = 0.0, f2 = 0.0;
    bool bad = false;
    tiled_force(a, s, i, own, f0, f1, f2, bad);
    if (own) {
        double* vi = a.v + ((int64_t)s * n + i) * 3;
        double v0 = vi[0], v1 = vi[1], v2 = vi[2];
        kick(v0, f0, a.max_f, a.dt);
        kick(v1, f1, a.max_f, a.dt);
        kick(v2, f2, a.max_f, a.dt);
        vi[0] = v0, vi[1] = v1, vi[2] = v2;
        if (bad) atomicCAS(reinterpret_cast<unsigned long long*>(a.status + s), ULLONG_MAX, (unsigned long long)t);
    }
}

// Step t, drift: x ← x + v·dt for every body of every system, then (slot >= 0) the state into frame slot.
__global__ void nbody_drift_kernel(const NbodyArgs a, const int64_t slot) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= (int64_t)a.S * a.n) return;
    double* xk = a.x + k * 3;
    const double* vk = a.v + k * 3;
    double x[3], v[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        v[d] = vk[d];
        x[d] = __dadd_rn(xk[d], __dmul_rn(v[d], a.dt));
        xk[d] = x[d];
    }
    if (slot >= 0) {
        const int64_t s = k / a.n, i = k % a.n;
        const int64_t f = ((s * a.R + slot) * a.n + i) * 3;
#pragma unroll
        for (int d = 0; d < 3; ++d) a.fx[f + d] = x[d], a.fv[f + d] = v[d];
    }
}

}  // namespace degnn

extern "C" {

int distegnn_nbody_simulate(int n_systems, int n_bodies, int64_t first_step, int64_t n_steps, int sample_freq,
                            double dt, double max_f, double* x, double* v, const double* q, double* frames_x,
                            double* frames_v, int64_t* status, void* stream) {
    using namespace degnn;
    DEGNN_CHECK_ARG(n_systems >= 0, "n_systems < 0");
    DEGNN_CHECK_ARG(n_bodies >= 2, "n_bodies < 2 (the force-size check needs an off-diagonal pair)");
    DEGNN_CHECK_ARG(first_step >= 0 && n_steps >= 0, "first_step or n_steps < 0");
    DEGNN_CHECK_ARG(sample_freq >= 1, "sample_freq < 1");
    DEGNN_CHECK_ARG(isfinite(dt) && !isnan(max_f), "dt not finite or max_f NaN");
    DEGNN_CHECK_ARG((int64_t)n_systems * n_bodies <= INT32_MAX, "n_systems * n_bodies >= 2^31");
    const int64_t end = first_step + n_steps;
    const int64_t k0 = (first_step + sample_freq - 1) / sample_freq;
    const int64_t R = end > 0 ? (end - 1) / sample_freq + 1 - k0 : 0;   // recorded t in [first_step, end)
    if (n_systems == 0 || n_steps == 0) return DISTEGNN_OK;
    DEGNN_CHECK_ARG(x && v && q && status, "null x, v, q or status");
    DEGNN_CHECK_ARG(R == 0 || (frames_x && frames_v), "null frames buffer and steps to record");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const NbodyArgs a{n_systems, n_bodies, R, dt, max_f, x, v, q, frames_x, frames_v, status};
    if (n_bodies <= NBODY_CTA_MAX) {
        const int per_cta = n_bodies < NBODY_CTA_PACK ? NBODY_CTA_PACK / n_bodies : 1;
        const int threads = (per_cta * n_bodies + 31) / 32 * 32;
        const int smem = per_cta * n_bodies * (int)(2 * sizeof(double2) + sizeof(double));
        const int blocks = (int)((n_systems + per_cta - 1) / per_cta);
        // one launch per recorded step: the steps after the previous recorded one, up to and including this one
        for (int64_t t = first_step; t < end;) {
            const int64_t rec = (t + sample_freq - 1) / sample_freq * sample_freq;
            const int64_t stop = rec < end ? rec + 1 : end;
            const int64_t slot = rec < end ? rec / sample_freq - k0 : -1;
            nbody_cta_kernel<<<blocks, threads, smem, st>>>(a, per_cta, t, (int)(stop - t), slot);   // <= sample_freq steps
            DEGNN_CHECK_LAUNCH();
            t = stop;
        }
    } else {
        const int nb = (n_bodies + NBODY_TILE - 1) / NBODY_TILE;
        DEGNN_CHECK_ARG((int64_t)n_systems * nb <= INT32_MAX, "too many CTAs");
        const int64_t total = (int64_t)n_systems * n_bodies;
        const int drift_threads = 256;
        const unsigned drift_blocks = (unsigned)((total + drift_threads - 1) / drift_threads);
        for (int64_t t = first_step; t < end; ++t) {
            nbody_force_tiled_kernel<<<n_systems * nb, NBODY_TILE, 0, st>>>(a, t);
            nbody_drift_kernel<<<drift_blocks, drift_threads, 0, st>>>(a, t % sample_freq == 0 ? t / sample_freq - k0 : -1);
            DEGNN_CHECK_LAUNCH();
        }
    }
    return DISTEGNN_OK;
}

}  // extern "C"

namespace degnn {

// ---- Sticks and hinges ------------------------------------------------------------------------------------------
// The reference's Stick.update and Hinge.update (physical_objects.py:101-145, 186-235), unit masses, in the fixed
// order of oracle/nbody_constrained_oracle.py: dot = (a0 b0 + a1 b1) + a2 b2, cross(a, b) = (a1 b2 − a2 b1, a2 b0 −
// a0 b2, a0 b1 − a1 b0), (M·r)_i = (M_i0 r0 + M_i1 r1) + M_i2 r2, no FMA, IEEE division and sqrt.  np.sin / np.cos
// become nbody_sincos and np.linalg.inv(A) @ a becomes solve3: the two places where numpy fixes no order.
struct d3 {
    double x, y, z;
};
__device__ __forceinline__ double dm(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double da(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ds(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ d3 add3(d3 a, d3 b) { return {da(a.x, b.x), da(a.y, b.y), da(a.z, b.z)}; }
__device__ __forceinline__ d3 sub3(d3 a, d3 b) { return {ds(a.x, b.x), ds(a.y, b.y), ds(a.z, b.z)}; }
__device__ __forceinline__ d3 mul3(d3 a, double s) { return {dm(a.x, s), dm(a.y, s), dm(a.z, s)}; }
__device__ __forceinline__ d3 div3(d3 a, double s) { return {__ddiv_rn(a.x, s), __ddiv_rn(a.y, s), __ddiv_rn(a.z, s)}; }
__device__ __forceinline__ double dot3(d3 a, d3 b) { return da(da(dm(a.x, b.x), dm(a.y, b.y)), dm(a.z, b.z)); }
__device__ __forceinline__ d3 cross3(d3 a, d3 b) {
    return {ds(dm(a.y, b.z), dm(a.z, b.y)), ds(dm(a.z, b.x), dm(a.x, b.z)), ds(dm(a.x, b.y), dm(a.y, b.x))};
}
// (M·r)_i for the rows m0, m1, m2 of M
__device__ __forceinline__ d3 matvec3(d3 m0, d3 m1, d3 m2, d3 r) { return {dot3(m0, r), dot3(m1, r), dot3(m2, r)}; }

// sin and cos of t: k = rint(t·2/π), the reduced argument t − k·π/2 as a double-double (hi, lo) from π/2 in three
// parts (k·C1 and k·C2 exact for |k| < 2^21), then minimax polynomials on [−π/4, π/4] (the published fdlibm
// coefficients) and the quadrant k mod 4.  Within 1 ulp of np.sin / np.cos for |t| <= 2^20 (beyond, k·C1 is inexact and
// accuracy degrades; non-finite t gives NaN).  oracle/nbody_constrained_oracle.py: sincos is the same sequence.
__device__ __noinline__ void nbody_sincos(const double t, double& sn, double& cs) {
    const double k = rint(dm(t, 6.36619772367581382433e-01));
    const double a = ds(t, dm(k, 1.57079632673412561417e+00));
    const double p2 = dm(k, 6.07710050630396597660e-11);
    const double hi1 = ds(a, p2);
    const double lo1 = ds(ds(a, hi1), p2);
    const double lo2 = ds(lo1, dm(k, 2.02226624879595063154e-21));
    const double x = da(hi1, lo2), y = da(ds(hi1, x), lo2);
    const double z = dm(x, x), w = dm(z, z);
    const double r = da(da(8.33333333332248946124e-03, dm(z, da(-1.98412698298579493134e-04, dm(z, 2.75573137070700676789e-06)))),
                        dm(dm(z, w), da(-2.50507602534068634195e-08, dm(z, 1.58969099521155010221e-10))));
    const double v = dm(z, x);
    const double s = ds(x, ds(ds(dm(z, ds(dm(0.5, y), dm(v, r))), y), dm(v, -1.66666666666666324348e-01)));
    const double rc = da(dm(z, da(4.16666666666666019037e-02,
                                  dm(z, da(-1.38888888888741095749e-03, dm(z, 2.48015872894767294178e-05))))),
                         dm(dm(w, w), da(-2.75573143513906633035e-07,
                                         dm(z, da(2.08757232129817482790e-09, dm(z, -1.13596475577881948265e-11))))));
    const double hz = dm(0.5, z), w1 = ds(1.0, hz);
    const double c = da(w1, da(ds(ds(1.0, w1), hz), ds(dm(z, rc), dm(x, y))));
    const double q = ds(k, dm(4.0, floor(dm(k, 0.25))));      // k mod 4, exact; NaN for a non-finite t
    if (q == 0.0) sn = s, cs = c;
    else if (q == 1.0) sn = c, cs = -s;
    else if (q == 2.0) sn = -s, cs = -c;
    else sn = -c, cs = s;
}

// get_rotation_matrix(|w|·dt, w/|w|)·r, the matrix entries as the reference writes them (physical_objects.py:10-24).
// w = 0 gives a 0/0 axis and NaN, as in numpy.
__device__ __forceinline__ d3 rotate(const d3 w, const d3 r, const double dt) {
    const double wn = __dsqrt_rn(dot3(w, w));
    const d3 d = div3(w, wn);
    double s, c;
    nbody_sincos(dm(wn, dt), s, c);
    const double oc = ds(1.0, c);
    const d3 m0 = {da(c, dm(dm(oc, d.x), d.x)), ds(dm(dm(oc, d.x), d.y), dm(s, d.z)), da(dm(dm(oc, d.x), d.z), dm(s, d.y))};
    const d3 m1 = {da(dm(dm(oc, d.x), d.y), dm(s, d.z)), da(c, dm(dm(oc, d.y), d.y)), ds(dm(dm(oc, d.y), d.z), dm(s, d.x))};
    const d3 m2 = {ds(dm(dm(oc, d.x), d.z), dm(s, d.y)), da(dm(dm(oc, d.y), d.z), dm(s, d.x)), da(c, dm(dm(oc, d.z), d.z))};
    return matvec3(m0, m1, m2, r);
}

// A⁻¹b by the adjugate: C_ij = A[i+1][j+1]·A[i+2][j+2] − A[i+1][j+2]·A[i+2][j+1] (indices mod 3), det = (A00 C00 +
// A01 C01) + A02 C02, x_i = ((C_0i b0 + C_1i b1) + C_2i b2) / det.  The hinge's A = I + e1e1ᵀ + e2e2ᵀ has eigenvalues
// in [1, 3], so det >= 1.
__device__ __forceinline__ d3 solve3(const double (&A)[3][3], const d3 b) {
    double C[3][3];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
            C[i][j] = ds(dm(A[i1][j1], A[i2][j2]), dm(A[i1][j2], A[i2][j1]));
        }
    const double det = da(da(dm(A[0][0], C[0][0]), dm(A[0][1], C[0][1])), dm(A[0][2], C[0][2]));
    const d3 x = {dot3({C[0][0], C[1][0], C[2][0]}, b), dot3({C[0][1], C[1][1], C[2][1]}, b),
                  dot3({C[0][2], C[1][2], C[2][2]}, b)};
    return div3(x, det);
}

// Stick.update: bodies (x0, f0), (x1, f1); st = (xc, vc, wc) read and written.  New x and v into x[], v[].
__device__ __noinline__ void stick_step(d3* x, d3* v, const d3 f0, const d3 f1, double* st, const double dt) {
    const d3 xc0 = {st[0], st[1], st[2]};
    d3 vc = {st[3], st[4], st[5]}, wc = {st[6], st[7], st[8]};
    const d3 r0 = sub3(x[0], xc0), r1 = sub3(x[1], xc0);
    const d3 ac = div3(add3(f0, f1), 2.0);
    vc = add3(vc, mul3(ac, dt));
    const d3 xc = add3(xc0, mul3(vc, dt));
    const double J = da(dot3(r0, r0), dot3(r1, r1));
    wc = add3(wc, mul3(div3(add3(cross3(r0, f0), cross3(r1, f1)), J), dt));
    const d3 _r0 = rotate(wc, r0, dt), _r1 = rotate(wc, r1, dt);
    x[0] = add3(xc, _r0), x[1] = add3(xc, _r1);
    v[0] = add3(vc, cross3(wc, _r0)), v[1] = add3(vc, cross3(wc, _r1));
    st[0] = xc.x, st[1] = xc.y, st[2] = xc.z, st[3] = vc.x, st[4] = vc.y, st[5] = vc.z;
    st[6] = wc.x, st[7] = wc.y, st[8] = wc.z;
}

// Hinge.update: bodies 0 (the joint), 1, 2 with forces f[]; st = (w1, w2) read and written.  New x and v into x[], v[].
__device__ __noinline__ void hinge_step(d3* x, d3* v, const d3* f, double* st, const double dt) {
    d3 w1 = {st[0], st[1], st[2]}, w2 = {st[3], st[4], st[5]};
    const d3 F = add3(add3(f[0], f[1]), f[2]);
    const d3 r01 = sub3(x[1], x[0]), r02 = sub3(x[2], x[0]);
    const d3 v01 = sub3(v[1], v[0]), v02 = sub3(v[2], v[0]);
    const double l1 = dot3(r01, r01), l2 = dot3(r02, r02);
    const d3 e1 = div3(r01, __dsqrt_rn(l1)), e2 = div3(r02, __dsqrt_rn(l2));
    const double ev1[3] = {e1.x, e1.y, e1.z}, ev2[3] = {e2.x, e2.y, e2.z};
    double A[3][3];
    d3 p1[3], p2[3];        // rows of I − e1e1ᵀ and I − e2e2ᵀ
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        double q1[3], q2[3];
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const double id = i == j ? 1.0 : 0.0, E1 = dm(ev1[i], ev1[j]), E2 = dm(ev2[i], ev2[j]);
            A[i][j] = da(da(id, E1), E2);
            q1[j] = ds(id, E1), q2[j] = ds(id, E2);
        }
        p1[i] = {q1[0], q1[1], q1[2]}, p2[i] = {q2[0], q2[1], q2[2]};
    }
    d3 a = sub3(sub3(F, cross3(w1, v01)), cross3(w2, v02));
    a = sub3(sub3(a, matvec3(p1[0], p1[1], p1[2], f[1])), matvec3(p2[0], p2[1], p2[2], f[2]));
    const d3 a0 = solve3(A, a);
    const d3 v0 = add3(v[0], mul3(a0, dt));
    const d3 x0 = add3(x[0], mul3(v0, dt));
    w1 = add3(w1, mul3(div3(cross3(r01, sub3(f[1], a0)), l1), dt));
    w2 = add3(w2, mul3(div3(cross3(r02, sub3(f[2], a0)), l2), dt));
    const d3 _r01 = rotate(w1, r01, dt), _r02 = rotate(w2, r02, dt);
    x[0] = x0, x[1] = add3(x0, _r01), x[2] = add3(x0, _r02);
    v[0] = v0, v[1] = add3(v0, cross3(w1, _r01)), v[2] = add3(v0, cross3(w2, _r02));
    st[0] = w1.x, st[1] = w1.y, st[2] = w1.z, st[3] = w2.x, st[4] = w2.y, st[5] = w2.z;
}

struct NbodyObjArgs {
    NbodyArgs a;
    int ns, nh;
    const int32_t *sticks, *hinges;     // [S, ns, 2], [S, nh, 3]
    double *sst, *hst;                  // [S, ns, 9], [S, nh, 6], read and written in place
    unsigned long long* invalid;        // += invalid table entries
    double* F;                          // n > 1024: clamped forces [S, n, 3] (workspace)
    int32_t* mark;                      // n > 1024: entries naming each body [S, n] (workspace)
    int32_t* sys_bad;                   // n > 1024: 1 where system s has an invalid entry [S] (workspace)
};

// Object u (< ns + nh) of system s: its kind, body count and table row.
struct ObjRef {
    bool stick;
    int nb;
    const int32_t* row;
    double* st;
};
__device__ __forceinline__ ObjRef obj_ref(const NbodyObjArgs& o, const int64_t s, const int u) {
    if (u < o.ns) return {true, 2, o.sticks + (s * o.ns + u) * 2, o.sst + (s * o.ns + u) * 9};
    const int h = u - o.ns;
    return {false, 3, o.hinges + (s * o.nh + h) * 3, o.hst + (s * o.nh + h) * 6};
}

// The object's entries that are out of [0, n) or name a body that another entry also names (mark: entries per body).
__device__ __forceinline__ int invalid_entries(const ObjRef& r, const int n, const int32_t* mark) {
    int bad = 0;
    for (int c = 0; c < r.nb; ++c) {
        const int b = r.row[c];
        bad += (b < 0 || b >= n) ? 1 : (mark[b] > 1);
    }
    return bad;
}

// One update of object r, whose bodies' state and clamped force the accessor B loads and stores.
template <class B>
__device__ __forceinline__ void object_step(const ObjRef& r, const B& bodies, const double dt) {
    d3 x[3], v[3], f[3];
    int b[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        b[c] = c < r.nb ? r.row[c] : r.row[0];
        x[c] = bodies.x(b[c]), v[c] = bodies.v(b[c]), f[c] = bodies.f(b[c]);
    }
    if (r.stick) stick_step(x, v, f[0], f[1], r.st, dt);
    else hinge_step(x, v, f, r.st, dt);
#pragma unroll
    for (int c = 0; c < 3; ++c)
        if (c < r.nb) bodies.store(b[c], x[c], v[c]);
}

// The CTA path's bodies of one system in shared memory: (x, y), (z, ‖x‖²), v, clamped F.
struct SmemBodies {
    double2 *pxy, *pzn;
    double *pv, *pf;
    __device__ d3 x(int j) const { return {pxy[j].x, pxy[j].y, pzn[j].x}; }
    __device__ d3 v(int j) const { return {pv[3 * j], pv[3 * j + 1], pv[3 * j + 2]}; }
    __device__ d3 f(int j) const { return {pf[3 * j], pf[3 * j + 1], pf[3 * j + 2]}; }
    __device__ void store(int j, d3 p, d3 u) const {
        pxy[j] = make_double2(p.x, p.y), pzn[j] = make_double2(p.z, norm2(p.x, p.y, p.z));
        pv[3 * j] = u.x, pv[3 * j + 1] = u.y, pv[3 * j + 2] = u.z;
    }
};

// The tiled path's bodies of one system in global memory: x, v [n, 3] and the clamped F of the workspace.
struct GmemBodies {
    double *px, *pv;
    const double* pf;
    __device__ d3 x(int j) const { return {px[3 * j], px[3 * j + 1], px[3 * j + 2]}; }
    __device__ d3 v(int j) const { return {pv[3 * j], pv[3 * j + 1], pv[3 * j + 2]}; }
    __device__ d3 f(int j) const { return {pf[3 * j], pf[3 * j + 1], pf[3 * j + 2]}; }
    __device__ void store(int j, d3 p, d3 u) const {
        px[3 * j] = p.x, px[3 * j + 1] = p.y, px[3 * j + 2] = p.z;
        pv[3 * j] = u.x, pv[3 * j + 1] = u.y, pv[3 * j + 2] = u.z;
    }
};

constexpr int NBODY_OBJ_SMEM = 2 * sizeof(double2) + 7 * sizeof(double) + sizeof(int32_t);    // per body, CTA path

// The CTA path with objects: as nbody_cta_kernel (systems blockIdx.x·per_cta .., thread k on body k of them, steps
// t0 .. t0 + steps − 1, then frame slot), with the whole state in shared memory.  Per step: every thread writes its
// body's clamped F; then thread i of a system updates body i if no object names it, and object i (stick i, then
// hinge i − ns) if i < ns + nh, each reading and writing only its own bodies.  The tables are checked at the start:
// a system with an out-of-range or repeated entry is not advanced, and with `count` its invalid entries are added to
// *invalid.  Shared memory: (x, y), (z, ‖x‖²), q, v, F and the entry count of every body of the CTA.
__global__ void __launch_bounds__(NBODY_CTA_MAX) nbody_obj_cta_kernel(const NbodyObjArgs o, const int per_cta,
                                                                      const int64_t t0, const int steps,
                                                                      const int64_t slot, const bool count) {
    extern __shared__ double2 sm[];
    const NbodyArgs& a = o.a;
    const int n = a.n, s0 = blockIdx.x * per_cta, G = min(per_cta, a.S - s0), k = threadIdx.x, P = per_cta * n;
    double2* sxy = sm;
    double2* szn = sm + P;
    double* sq = reinterpret_cast<double*>(sm + 2 * P);
    double* sv = sq + P;
    double* sf = sv + 3 * P;
    int32_t* smark = reinterpret_cast<int32_t*>(sf + 3 * P);
    __shared__ unsigned long long first_bad[NBODY_CTA_PACK / 2];
    __shared__ int sys_bad[NBODY_CTA_PACK / 2];
    const bool own = k < G * n;
    const int g = k / n, i = k - g * n, s = s0 + g;
    const int64_t row = ((int64_t)s0 * n + k) * 3;
    if (own) {
        const double x0 = a.x[row], x1 = a.x[row + 1], x2 = a.x[row + 2];
        sxy[k] = make_double2(x0, x1);
        szn[k] = make_double2(x2, norm2(x0, x1, x2));
        sv[3 * k] = a.v[row], sv[3 * k + 1] = a.v[row + 1], sv[3 * k + 2] = a.v[row + 2];
        sq[k] = a.q[(int64_t)s0 * n + k];
    }
    if (k < P) smark[k] = 0;
    if (k < per_cta) first_bad[k] = ULLONG_MAX, sys_bad[k] = 0;
    __syncthreads();
    const bool obj = own && i < o.ns + o.nh;
    ObjRef r{};
    if (obj) {
        r = obj_ref(o, s, i);
        for (int c = 0; c < r.nb; ++c) {
            const int b = r.row[c];
            if (b >= 0 && b < n) atomicAdd(&smark[g * n + b], 1);
        }
    }
    __syncthreads();
    if (obj) {
        const int bad = invalid_entries(r, n, smark + g * n);
        if (bad) {
            sys_bad[g] = 1;
            if (count) atomicAdd(o.invalid, (unsigned long long)bad);
        }
    }
    __syncthreads();
    const bool live = own && !sys_bad[g];
    const bool iso = live && smark[k] == 0;
    const SmemBodies bodies{sxy + g * n, szn + g * n, sv + g * n * 3, sf + g * n * 3};
    const double2* gxy = sxy + g * n;
    const double2* gzn = szn + g * n;
    const double* gq = sq + g * n;
    unsigned long long my_bad = ULLONG_MAX;
    for (int u = 0; u < steps; ++u) {
        if (own) {
            const double2 xy = sxy[k], zn = szn[k];
            double f0 = 0.0, f1 = 0.0, f2 = 0.0;
            bool bad = false;
            for (int j = 0; j < n; ++j) {
                const double2 pxy = gxy[j], pzn = gzn[j];
                pair_term(xy.x, xy.y, zn.x, zn.y, sq[k], pxy.x, pxy.y, pzn.x, pzn.y, gq[j], j == i, f0, f1, f2, bad);
            }
            if (bad && my_bad == ULLONG_MAX) my_bad = (unsigned long long)(t0 + u);
            sf[3 * k] = clamp_f(f0, a.max_f), sf[3 * k + 1] = clamp_f(f1, a.max_f), sf[3 * k + 2] = clamp_f(f2, a.max_f);
        }
        __syncthreads();        // every F is written and every read of this step's positions is done
        if (iso) {              // v ← v + F·dt, x ← x + v·dt
            const d3 v = add3(bodies.v(i), mul3(bodies.f(i), a.dt));
            bodies.store(i, add3(bodies.x(i), mul3(v, a.dt)), v);
        }
        if (live && obj) object_step(r, bodies, a.dt);
        __syncthreads();        // the new state is in place before the next step reads it
    }
    if (my_bad != ULLONG_MAX) atomicMin(&first_bad[g], my_bad);
    if (own) {
        const double2 xy = sxy[k], zn = szn[k];
        const double v0 = sv[3 * k], v1 = sv[3 * k + 1], v2 = sv[3 * k + 2];
        a.x[row] = xy.x, a.x[row + 1] = xy.y, a.x[row + 2] = zn.x;
        a.v[row] = v0, a.v[row + 1] = v1, a.v[row + 2] = v2;
        if (slot >= 0) {
            const int64_t f = (((int64_t)s * a.R + slot) * n + i) * 3;
            a.fx[f] = xy.x, a.fx[f + 1] = xy.y, a.fx[f + 2] = zn.x;
            a.fv[f] = v0, a.fv[f + 1] = v1, a.fv[f + 2] = v2;
        }
    }
    __syncthreads();
    if (k < G && first_bad[k] != ULLONG_MAX && a.status[s0 + k] < 0) a.status[s0 + k] = (int64_t)first_bad[k];
}

// Tiled path, once per call: o.mark[s, b] = entries naming body b (o.mark zeroed before), thread per (system, object).
__global__ void nbody_obj_mark_kernel(const NbodyObjArgs o) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, m = o.ns + o.nh;
    if (k >= (int64_t)o.a.S * m) return;
    const int64_t s = k / m;
    const ObjRef r = obj_ref(o, s, (int)(k - s * m));
    for (int c = 0; c < r.nb; ++c) {
        const int b = r.row[c];
        if (b >= 0 && b < o.a.n) atomicAdd(&o.mark[s * o.a.n + b], 1);
    }
}

// Tiled path, once per call: invalid entries into *o.invalid and o.sys_bad (zeroed before).
__global__ void nbody_obj_check_kernel(const NbodyObjArgs o) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, m = o.ns + o.nh;
    if (k >= (int64_t)o.a.S * m) return;
    const int64_t s = k / m;
    const int bad = invalid_entries(obj_ref(o, s, (int)(k - s * m)), o.a.n, o.mark + s * o.a.n);
    if (bad) {
        o.sys_bad[s] = 1;
        atomicAdd(o.invalid, (unsigned long long)bad);
    }
}

// Tiled path, step t: the clamped F of every body into the workspace (no kick), status as nbody_force_tiled_kernel.
__global__ void __launch_bounds__(NBODY_TILE) nbody_obj_force_tiled_kernel(const NbodyObjArgs o, const int64_t t) {
    const int n = o.a.n, nb = (n + NBODY_TILE - 1) / NBODY_TILE;
    const int s = blockIdx.x / nb, i = (blockIdx.x % nb) * NBODY_TILE + threadIdx.x;
    const bool own = i < n;
    double f0 = 0.0, f1 = 0.0, f2 = 0.0;
    bool bad = false;
    tiled_force(o.a, s, i, own, f0, f1, f2, bad);
    if (own) {
        double* fi = o.F + ((int64_t)s * n + i) * 3;
        fi[0] = clamp_f(f0, o.a.max_f), fi[1] = clamp_f(f1, o.a.max_f), fi[2] = clamp_f(f2, o.a.max_f);
        if (bad) atomicCAS(reinterpret_cast<unsigned long long*>(o.a.status + s), ULLONG_MAX, (unsigned long long)t);
    }
}

// Tiled path, step t, the update: thread (s, u) for u < n takes body u when no object names it (kick and drift), for
// u >= n object u − n; then (slot >= 0) the bodies it updated into frame slot.  A system with an invalid entry is not
// advanced; its body threads record every body.
__global__ void nbody_obj_update_kernel(const NbodyObjArgs o, const int64_t slot) {
    const NbodyArgs& a = o.a;
    const int n = a.n, m = n + o.ns + o.nh;
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= (int64_t)a.S * m) return;
    const int64_t s = k / m;
    const int u = (int)(k - s * m);
    const bool live = !o.sys_bad[s];
    const GmemBodies bodies{a.x + s * n * 3, a.v + s * n * 3, o.F + s * n * 3};
    int b[3] = {u, u, u}, nb = 0;
    if (u < n) {
        if (!live || o.mark[s * n + u] == 0) nb = 1;
        if (live && nb) {
            const d3 v = add3(bodies.v(u), mul3(bodies.f(u), a.dt));
            bodies.store(u, add3(bodies.x(u), mul3(v, a.dt)), v);
        }
    } else if (live) {
        const ObjRef r = obj_ref(o, s, u - n);
        object_step(r, bodies, a.dt);
        nb = r.nb;
#pragma unroll
        for (int c = 0; c < 3; ++c)
            if (c < nb) b[c] = r.row[c];
    }
    if (slot < 0) return;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        if (c >= nb) break;
        const int64_t f = ((s * a.R + slot) * n + b[c]) * 3;
        const d3 x = bodies.x(b[c]), v = bodies.v(b[c]);
        a.fx[f] = x.x, a.fx[f + 1] = x.y, a.fx[f + 2] = x.z;
        a.fv[f] = v.x, a.fv[f + 1] = v.y, a.fv[f + 2] = v.z;
    }
}

int64_t nbody_obj_workspace(int64_t S, int64_t n) {
    if (n <= NBODY_CTA_MAX) return 0;
    WorkspaceCursor w;
    w.take(S * n * 3 * sizeof(double));
    w.take(S * n * sizeof(int32_t));
    w.take(S * sizeof(int32_t));
    return (int64_t)w.end;
}


}  // namespace degnn

extern "C" {

int distegnn_nbody_objects_workspace_bytes(int n_systems, int n_bodies, int64_t* bytes) {
    using namespace degnn;
    DEGNN_CHECK_ARG(bytes, "null output pointer");
    DEGNN_CHECK_ARG(n_systems >= 0 && n_bodies >= 0, "negative size");
    *bytes = nbody_obj_workspace(n_systems, n_bodies);
    return DISTEGNN_OK;
}

int distegnn_nbody_simulate_objects(int n_systems, int n_bodies, int n_sticks, int n_hinges, int64_t first_step,
                                    int64_t n_steps, int sample_freq, double dt, double max_f, double* x, double* v,
                                    const double* q, const int32_t* sticks, const int32_t* hinges,
                                    double* stick_state, double* hinge_state, double* frames_x, double* frames_v,
                                    int64_t* status, int64_t* invalid, void* workspace, int64_t workspace_bytes,
                                    void* stream) {
    using namespace degnn;
    DEGNN_CHECK_ARG(n_systems >= 0, "n_systems < 0");
    DEGNN_CHECK_ARG(n_sticks >= 0 && n_hinges >= 0, "n_sticks or n_hinges < 0");
    DEGNN_CHECK_ARG(n_sticks + n_hinges >= 1, "no sticks or hinges (distegnn_nbody_simulate runs isolated bodies)");
    DEGNN_CHECK_ARG(n_bodies >= 2 * (int64_t)n_sticks + 3 * (int64_t)n_hinges,
                    "n_bodies < 2 * n_sticks + 3 * n_hinges (the objects' bodies must be distinct)");
    DEGNN_CHECK_ARG(first_step >= 0 && n_steps >= 0, "first_step or n_steps < 0");
    DEGNN_CHECK_ARG(sample_freq >= 1, "sample_freq < 1");
    DEGNN_CHECK_ARG(isfinite(dt) && !isnan(max_f), "dt not finite or max_f NaN");
    DEGNN_CHECK_ARG((int64_t)n_systems * (n_bodies + n_sticks + n_hinges) <= INT32_MAX,
                    "n_systems * (n_bodies + n_sticks + n_hinges) >= 2^31");
    const int64_t end = first_step + n_steps;
    const int64_t k0 = (first_step + sample_freq - 1) / sample_freq;
    const int64_t R = end > 0 ? (end - 1) / sample_freq + 1 - k0 : 0;   // recorded t in [first_step, end)
    if (n_systems == 0 || n_steps == 0) return DISTEGNN_OK;
    DEGNN_CHECK_ARG(x && v && q && status && invalid, "null x, v, q, status or invalid");
    DEGNN_CHECK_ARG(n_sticks == 0 || (sticks && stick_state), "null sticks or stick_state");
    DEGNN_CHECK_ARG(n_hinges == 0 || (hinges && hinge_state), "null hinges or hinge_state");
    DEGNN_CHECK_ARG(R == 0 || (frames_x && frames_v), "null frames buffer and steps to record");
    const int64_t need = nbody_obj_workspace(n_systems, n_bodies);
    if (workspace_bytes < need || (need > 0 && !workspace)) {
        set_error("distegnn_nbody_simulate_objects: workspace %lld < %lld bytes", (long long)workspace_bytes,
                  (long long)need);
        return DISTEGNN_EWORKSPACE;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    NbodyObjArgs o{{n_systems, n_bodies, R, dt, max_f, x, v, q, frames_x, frames_v, status}, n_sticks, n_hinges, sticks,
                   hinges, stick_state, hinge_state, reinterpret_cast<unsigned long long*>(invalid), nullptr, nullptr,
                   nullptr};
    if (n_bodies <= NBODY_CTA_MAX) {
        const int per_cta = n_bodies < NBODY_CTA_PACK ? NBODY_CTA_PACK / n_bodies : 1;
        const int threads = (per_cta * n_bodies + 31) / 32 * 32;
        const int smem = per_cta * n_bodies * NBODY_OBJ_SMEM;
        const int blocks = (int)((n_systems + per_cta - 1) / per_cta);
        ensure_dynamic_smem((const void*)nbody_obj_cta_kernel, NBODY_CTA_MAX * NBODY_OBJ_SMEM);
        for (int64_t t = first_step; t < end;) {
            const int64_t rec = (t + sample_freq - 1) / sample_freq * sample_freq;
            const int64_t stop = rec < end ? rec + 1 : end;
            const int64_t slot = rec < end ? rec / sample_freq - k0 : -1;
            nbody_obj_cta_kernel<<<blocks, threads, smem, st>>>(o, per_cta, t, (int)(stop - t), slot, t == first_step);
            DEGNN_CHECK_LAUNCH();
            t = stop;
        }
    } else {
        const int nb = (n_bodies + NBODY_TILE - 1) / NBODY_TILE;
        DEGNN_CHECK_ARG((int64_t)n_systems * nb <= INT32_MAX, "too many CTAs");
        WorkspaceCursor w;
        char* base = static_cast<char*>(workspace);
        o.F = reinterpret_cast<double*>(base + w.take((int64_t)n_systems * n_bodies * 3 * sizeof(double)));
        o.mark = reinterpret_cast<int32_t*>(base + w.take((int64_t)n_systems * n_bodies * sizeof(int32_t)));
        o.sys_bad = reinterpret_cast<int32_t*>(base + w.take((int64_t)n_systems * sizeof(int32_t)));
        const int threads = 256;
        cudaMemsetAsync(o.mark, 0, (size_t)(reinterpret_cast<char*>(o.sys_bad) - reinterpret_cast<char*>(o.mark)) +
                                       (size_t)n_systems * sizeof(int32_t), st);
        const int64_t n_obj = (int64_t)n_systems * (n_sticks + n_hinges);
        const unsigned obj_blocks = (unsigned)((n_obj + threads - 1) / threads);
        nbody_obj_mark_kernel<<<obj_blocks, threads, 0, st>>>(o);
        nbody_obj_check_kernel<<<obj_blocks, threads, 0, st>>>(o);
        DEGNN_CHECK_LAUNCH();
        const unsigned upd_blocks =
            (unsigned)(((int64_t)n_systems * (n_bodies + n_sticks + n_hinges) + threads - 1) / threads);
        for (int64_t t = first_step; t < end; ++t) {
            nbody_obj_force_tiled_kernel<<<n_systems * nb, NBODY_TILE, 0, st>>>(o, t);
            nbody_obj_update_kernel<<<upd_blocks, threads, 0, st>>>(o, t % sample_freq == 0 ? t / sample_freq - k0 : -1);
            DEGNN_CHECK_LAUNCH();
        }
    }
    return DISTEGNN_OK;
}

}  // extern "C"
