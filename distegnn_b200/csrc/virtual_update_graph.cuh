// Body of the virtual-node update of graph `b` by one CTA of VU_THREADS threads (virtual_update.cu), included INSIDE a
// kernel's body: by virtual_update_kernel<SYNC> and by the testing library's W-rank twin (testing/comm_ranks.cu).  The
// including kernel defines `SYNC` (bool), `a` (VUpdArgs), `cd` (CommDev), `b` (graph) and `pause` (passed to
// comm_slot_allreduce).  It is a fragment rather than a __forceinline__ function because the call boundary, inlined or
// not, changes the register allocation of virtual_update_kernel<true>: with a fragment the product's SASS is the code it
// had before the twin existed.  No include guard: one inclusion per kernel.
    constexpr int MC = DISTEGNN_MAX_CHANNELS;
    __shared__ float sV[VU_KMAX];       // vsum[b,:] (summed over the partitions)
    __shared__ float sX[3 * MC];        // new Xv [3][C]
    __shared__ float sZ[3 * MC];        // Xv − x̄
    __shared__ float sM[MC * MC];       // m_X
    __shared__ float sHv[MC * H];       // Hv (old, then new) [C][64]
    __shared__ float sAg[MC * H];       // mean mv [C][64]
    __shared__ float sT[MC * H];        // hidden of node_mlp_virtual
    const int tid = threadIdx.x, C = a.C;
    float* vg = a.vsum + (size_t)b * a.K;
    const bool init = a.flags & DISTEGNN_FLAG_INIT;
    const bool last = a.flags & DISTEGNN_FLAG_LAST;
    const bool zero = a.flags & DISTEGNN_FLAG_ZERO_VSUM;
    for (int i = tid; i < a.K; i += VU_THREADS) sV[i] = vg[i];
    __syncthreads();
    if (SYNC) comm_slot_allreduce(cd, b, sV, a.K, pause);
    if (zero) {
        for (int i = tid; i < a.K; i += VU_THREADS) vg[i] = 0.f;
    } else if (SYNC) {
        for (int i = tid; i < a.K; i += VU_THREADS) vg[i] = sV[i];
    }
    const float* vs = sV;
    const float inv = 1.0f / fmaxf(vs[3], 1.0f);

    if (tid < 3 * C) {
        float x;
        if (init && (a.flags & DISTEGNN_FLAG_INIT_CENTROID)) x = vs[tid / C] * inv;   // X_0 = x̄ of these positions
        else x = (init && a.init_loc_mean) ? a.init_loc_mean[(size_t)b * 3 + tid / C] : a.Xv[(size_t)b * 3 * C + tid];
        if (!init) x += vs[4 + tid] * inv;
        sX[tid] = x;
        a.Xv[(size_t)b * 3 * C + tid] = x;
        sZ[tid] = x - vs[tid / C] * inv;   // tid / C = spatial dim
    }
    if (last) return;
    for (int i = tid; i < C * H; i += VU_THREADS) {
        const float hv = (init && a.init_hv0) ? a.init_hv0[i] : a.Hv[(size_t)b * C * H + i];
        sHv[i] = hv;
        if (init && a.init_hv0) a.Hv[(size_t)b * C * H + i] = hv;
        sAg[i] = init ? 0.f : vs[4 + 3 * C + i] * inv;
    }
    __syncthreads();
    if (tid < C * C) {
        const int i = tid / C, j = tid - i * C;
        sM[tid] = sZ[i] * sZ[j] + sZ[C + i] * sZ[C + j] + sZ[2 * C + i] * sZ[2 * C + j];
    }
    if (!init) {
        // Hv' = Hv + W2·SiLU(W1·[Hv; agg] + b1) + b2   (per channel; thread per (c, n))
        for (int i = tid; i < C * H; i += VU_THREADS) {
            const int c = i / H, n = i - c * H;
            float s = __ldg(a.mb1 + n);
            // weights come straight from L2 (each is used by C rows only); the 64-step loops are fully unrolled by the
            // compiler, i.e. all loads of a row are in flight together
            for (int k = 0; k < H; ++k) s = fmaf(sHv[c * H + k], __ldg(a.m1 + k * H + n), s);
            for (int k = 0; k < H; ++k) s = fmaf(sAg[c * H + k], __ldg(a.m1 + (H + k) * H + n), s);
            sT[i] = silu(s);
        }
        __syncthreads();
        float upd[(MC * H + VU_THREADS - 1) / VU_THREADS];
        int u = 0;
        for (int i = tid; i < C * H; i += VU_THREADS, ++u) {
            const int c = i / H, n = i - c * H;
            float s = __ldg(a.mb2 + n);
            for (int k = 0; k < H; ++k) s = fmaf(sT[c * H + k], __ldg(a.m2 + k * H + n), s);
            upd[u] = sHv[i] + s;
        }
        __syncthreads();
        u = 0;
        for (int i = tid; i < C * H; i += VU_THREADS, ++u) {
            sHv[i] = upd[u];
            a.Hv[(size_t)b * C * H + i] = upd[u];
        }
    }
    __syncthreads();
    // G[c][n] = Σ_k W1v_V[k][n]·Hv'[c][k] + Σ_j W1v_M[j][n]·m_X[j][c] + b1v[n]
    for (int i = tid; i < C * H; i += VU_THREADS) {
        const int c = i / H, n = i - c * H;
        float s = __ldg(a.nvb1 + n);
        for (int k = 0; k < H; ++k) s = fmaf(sHv[c * H + k], __ldg(a.nv1v + k * H + n), s);
        for (int j = 0; j < C; ++j) s = fmaf(sM[j * C + c], __ldg(a.nv1m + j * H + n), s);
        a.G[(size_t)b * C * H + i] = s;
    }
