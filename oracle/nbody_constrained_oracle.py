"""Float64 numpy restatement of the constrained N-body step of distegnn_b200.nbody (sticks and hinges, DESIGN §25) in its
fixed arithmetic order: the bits csrc/nbody.cu's object kernels must reproduce.  The force is nbody_oracle.forces,
clamped; isolated bodies then take v ← v + F·dt, x ← x + v·dt, and each stick and hinge restates the reference's
`Stick.update` / `Hinge.update` (physical_objects.py) with

  dot(a, b) = (a0 b0 + a1 b1) + a2 b2,  cross(a, b) = (a1 b2 − a2 b1, a2 b0 − a0 b2, a0 b1 − a1 b0),
  M·r = ((M_i0 r0 + M_i1 r1) + M_i2 r2)_i,

every product and sum rounded on its own (numpy's elementwise ufuncs: no FMA), IEEE division and sqrt, and two
choices of its own where numpy fixes no order:
  sincos    Cody–Waite reduction by π/2 and the fixed polynomials below (instead of np.sin / np.cos)
  solve3    A⁻¹a as adj(A)·a / det(A), cofactors in the cyclic form (instead of np.linalg.inv(A) @ a)
Vectorised over systems and objects."""
from __future__ import annotations

import numpy as np

from oracle import nbody_oracle

# π/2 in three parts: C1 (31 significant bits) and C2 (32) so that k·C1 and k·C2 are exact for |k| < 2^21, and C3
# the rest (their sum is π/2 within 1e-37); 2/π rounded
INV_PIO2 = 6.36619772367581382433e-01
PIO2_1, PIO2_2, PIO2_3 = 1.57079632673412561417e+00, 6.07710050630396597660e-11, 2.02226624879595063154e-21
SINCOS_RANGE = 2.0 ** 20        # |θ| up to here: the reduction is exact to ~2^-100 relative (see sincos)
# minimax polynomials of sin and cos on [−π/4, π/4] (the published fdlibm coefficients)
S1, S2, S3 = -1.66666666666666324348e-01, 8.33333333332248946124e-03, -1.98412698298579493134e-04
S4, S5, S6 = 2.75573137070700676789e-06, -2.50507602534068634195e-08, 1.58969099521155010221e-10
K1, K2, K3 = 4.16666666666666019037e-02, -1.38888888888741095749e-03, 2.48015872894767294178e-05
K4, K5, K6 = -2.75573143513906633035e-07, 2.08757232129817482790e-09, -1.13596475577881948265e-11


def _kernel_sin(x, y):
    # sin(x + y) for |x| <= π/4, |y| <= ulp(x)/2
    z = x * x
    w = z * z
    r = (S2 + z * (S3 + z * S4)) + (z * w) * (S5 + z * S6)
    v = z * x
    return x - (((z * (0.5 * y - v * r)) - y) - v * S1)


def _kernel_cos(x, y):
    z = x * x
    w = z * z
    r = z * (K1 + z * (K2 + z * K3)) + (w * w) * (K4 + z * (K5 + z * K6))
    hz = 0.5 * z
    w = 1.0 - hz
    return w + (((1.0 - w) - hz) + (z * r - x * y))


def sincos(theta):
    """(sin θ, cos θ), elementwise.  k = rint(θ·2/π); the reduced argument r = θ − k·π/2 is kept as a double-double
    (hi, lo): a = θ − k·C1 (exact), hi1 = a − k·C2 with its exact rounding error, lo folds in −k·C3, and one Fast2Sum
    renormalises.  Then the polynomials at (hi, lo) and the quadrant k mod 4.  Within 1 ulp of np.sin / np.cos for
    |θ| <= SINCOS_RANGE (tests/test_nbody_constrained.py); beyond it k·C1 is no longer exact and the result loses
    accuracy (still the same bits here and on the device, csrc/nbody.cu: nbody_sincos); ±inf and NaN give NaN."""
    t = np.asarray(theta, dtype=np.float64)
    with np.errstate(all="ignore"):
        k = np.rint(t * INV_PIO2)
        a = t - k * PIO2_1
        p2 = k * PIO2_2
        hi1 = a - p2
        lo1 = (a - hi1) - p2
        lo = lo1 - k * PIO2_3
        hi = hi1 + lo
        lo = (hi1 - hi) + lo
        s, c = _kernel_sin(hi, lo), _kernel_cos(hi, lo)
        q = k - 4.0 * np.floor(k * 0.25)            # k mod 4, exact; NaN for a non-finite θ
    sin = np.where(q == 0, s, np.where(q == 1, c, np.where(q == 2, -s, -c)))
    cos = np.where(q == 0, c, np.where(q == 1, -s, np.where(q == 2, -c, s)))
    return sin, cos


def dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], axis=-1)


def matvec(M, r):
    return (M[..., 0] * r[..., None, 0] + M[..., 1] * r[..., None, 1]) + M[..., 2] * r[..., None, 2]


def solve3(A, b):
    """A⁻¹b for A [...,3,3], b [...,3]: C_ij = A[i+1][j+1]·A[i+2][j+2] − A[i+1][j+2]·A[i+2][j+1] (indices mod 3),
    det = (A00 C00 + A01 C01) + A02 C02, x_i = ((C_0i b0 + C_1i b1) + C_2i b2) / det."""
    C = np.empty_like(A)
    for i in range(3):
        for j in range(3):
            i1, i2, j1, j2 = (i + 1) % 3, (i + 2) % 3, (j + 1) % 3, (j + 2) % 3
            C[..., i, j] = A[..., i1, j1] * A[..., i2, j2] - A[..., i1, j2] * A[..., i2, j1]
    det = (A[..., 0, 0] * C[..., 0, 0] + A[..., 0, 1] * C[..., 0, 1]) + A[..., 0, 2] * C[..., 0, 2]
    x = (C[..., 0, :] * b[..., None, 0] + C[..., 1, :] * b[..., None, 1]) + C[..., 2, :] * b[..., None, 2]
    return x / det[..., None]


def rotate(w, r, dt):
    """The reference's get_rotation_matrix(|w|·dt, w / |w|) applied to r, entry by entry as it writes them."""
    wn = np.sqrt(dot(w, w))
    d = w / wn[..., None]
    s, c = sincos(wn * dt)
    x, y, z = d[..., 0], d[..., 1], d[..., 2]
    oc = 1.0 - c
    M = np.stack([
        np.stack([c + oc * x * x, oc * x * y - s * z, oc * x * z + s * y], -1),
        np.stack([oc * x * y + s * z, c + oc * y * y, oc * y * z - s * x], -1),
        np.stack([oc * x * z - s * y, oc * y * z + s * x, c + oc * z * z], -1)], -2)
    return matvec(M, r)


def stick_update(x, v, F, idx, st, dt):
    """Stick.update of every stick: x, v [S,n,3] updated in place at the table's bodies idx [S,ns,2]; st [S,ns,9]
    (xc, vc, wc) returned updated."""
    S = np.arange(x.shape[0])[:, None]
    b0, b1 = idx[..., 0], idx[..., 1]
    x0, x1, f0, f1 = x[S, b0], x[S, b1], F[S, b0], F[S, b1]
    xc, vc, wc = st[..., 0:3], st[..., 3:6], st[..., 6:9]
    r0, r1 = x0 - xc, x1 - xc
    ac = (f0 + f1) / 2.0
    vc = vc + ac * dt
    xc = xc + vc * dt
    J = dot(r0, r0) + dot(r1, r1)
    beta = (cross(r0, f0) + cross(r1, f1)) / J[..., None]
    wc = wc + beta * dt
    _r0, _r1 = rotate(wc, r0, dt), rotate(wc, r1, dt)
    x[S, b0], x[S, b1] = xc + _r0, xc + _r1
    v[S, b0], v[S, b1] = vc + cross(wc, _r0), vc + cross(wc, _r1)
    return np.concatenate([xc, vc, wc], -1)


def hinge_update(x, v, F, idx, st, dt):
    """Hinge.update of every hinge: x, v updated in place at idx [S,nh,3]; st [S,nh,6] (w1, w2) returned updated."""
    S = np.arange(x.shape[0])[:, None]
    b0, b1, b2 = idx[..., 0], idx[..., 1], idx[..., 2]
    x0, x1, x2, v0, v1, v2 = x[S, b0], x[S, b1], x[S, b2], v[S, b0], v[S, b1], v[S, b2]
    f0, f1, f2 = F[S, b0], F[S, b1], F[S, b2]
    w1, w2 = st[..., 0:3], st[..., 3:6]
    f = (f0 + f1) + f2
    r01, r02 = x1 - x0, x2 - x0
    v01, v02 = v1 - v0, v2 - v0
    e1 = r01 / np.sqrt(dot(r01, r01))[..., None]
    e2 = r02 / np.sqrt(dot(r02, r02))[..., None]
    E1 = e1[..., :, None] * e1[..., None, :]
    E2 = e2[..., :, None] * e2[..., None, :]
    I = np.eye(3)
    A = (I + E1) + E2
    a = (f - cross(w1, v01)) - cross(w2, v02)
    a = (a - matvec(I - E1, f1)) - matvec(I - E2, f2)
    a0 = solve3(A, a)
    v0 = v0 + a0 * dt
    x0 = x0 + v0 * dt
    w1 = w1 + (cross(r01, f1 - a0) / dot(r01, r01)[..., None]) * dt
    w2 = w2 + (cross(r02, f2 - a0) / dot(r02, r02)[..., None]) * dt
    _r01, _r02 = rotate(w1, r01, dt), rotate(w2, r02, dt)
    x[S, b0], x[S, b1], x[S, b2] = x0, x0 + _r01, x0 + _r02
    v[S, b0], v[S, b1], v[S, b2] = v0, v0 + cross(w1, _r01), v0 + cross(w2, _r02)
    return np.concatenate([w1, w2], -1)


def simulate(x0, v0, q, sticks, hinges, stick_state, hinge_state, n_steps: int, sample_freq: int = 100,
             dt: float = 1e-3, first_step: int = 0, status=None):
    """n_steps steps first_step .. of the systems (x0, v0 [S,n,3], q [S,n] or [S,n,1]) with the object tables sticks
    [S,ns,2], hinges [S,nh,3] and states stick_state [S,ns,9], hinge_state [S,nh,6].  Returns (x, v, frames_x,
    frames_v [S,R,n,3], status [S], stick_state, hinge_state), as nbody_oracle.simulate plus the object states."""
    x, v = np.array(x0, dtype=np.float64), np.array(v0, dtype=np.float64)
    S, n = x.shape[0], x.shape[1]
    q = np.asarray(q, dtype=np.float64).reshape(S, -1)
    sticks = np.asarray(sticks, dtype=np.int64).reshape(S, -1, 2)
    hinges = np.asarray(hinges, dtype=np.int64).reshape(S, -1, 3)
    ss = np.array(stick_state, dtype=np.float64).reshape(S, -1, 9)
    hs = np.array(hinge_state, dtype=np.float64).reshape(S, -1, 6)
    iso = np.ones((S, n), dtype=bool)
    for tab in (sticks, hinges):
        for c in range(tab.shape[2]):
            iso[np.arange(S)[:, None], tab[..., c]] = False
    st = np.full(S, -1, dtype=np.int64) if status is None else np.array(status, dtype=np.int64)
    max_f = 0.1 / dt
    fx, fv = [], []
    with np.errstate(all="ignore"):
        for t in range(first_step, first_step + n_steps):
            F, bad = nbody_oracle.forces(x, q)
            st[(st < 0) & bad] = t
            F = np.where(F > max_f, max_f, np.where(F < -max_f, -max_f, F))
            xn, vn = x.copy(), v.copy()
            vi = v + F * dt
            xn[iso], vn[iso] = (x + vi * dt)[iso], vi[iso]
            if sticks.shape[1]:
                ss = stick_update(xn, vn, F, sticks, ss, dt)
            if hinges.shape[1]:
                hs = hinge_update(xn, vn, F, hinges, hs, dt)
            x, v = xn, vn
            if t % sample_freq == 0:
                fx.append(x.copy())
                fv.append(v.copy())
    shape = (S, 0) + x.shape[1:]
    stack = lambda a: np.stack(a, axis=1) if a else np.zeros(shape)
    return x, v, stack(fx), stack(fv), st, ss, hs
