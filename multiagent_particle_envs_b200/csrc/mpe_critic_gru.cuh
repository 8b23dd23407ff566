// mpe_critic_gru.cuh -- one evaluation and the value store of rMAPPO's recurrent centralized critic (RCriticArgs,
// RCriticShape in mpe_kernels.cu), shared by the one shared critic (mpe_critic_gru.cu), the per-agent critics of the
// separated runner (mpe_gru_separated.cu) and IPPO's recurrent local critic (mpe_critic_local.cu).  Included after mpe_kernels.cu's templates.
#pragma once

namespace mpe {

// One evaluation of the critic for the warp's m-tile (rows g and g + 8 of this lane are worlds wa and wb): x =
// base(share_obs), h' = GRU(x, h) into hn, and V(LN(h')) into v (column 0 of rows g and g + 8 in elements 0 and 2 of
// the quad's first lane).  src[i] points at agent i's [n][obs_dim_i] observations of the step.  The input LayerNorm's
// fp32 two-pass statistics over all D entries come from the A fragments themselves (a row's entries are spread over
// the 4 lanes of a quad); the records are then read a third time, normalised, rounded to TF32 and multiplied by agent
// i's k-tiles of W1.  Layers 2 and 3 are MAPPO's (act_norm_tf32_frags), the cell the recurrent actor's (gru_cell).
// K >= 0: IPPO's local critic on agent K's columns alone (RCriticShape<P, K>), src[K] its observations.
template <class P, int K = -1>
__device__ __forceinline__ void rcritic_eval(const float *__restrict__ Wsm, const float *const (&src)[P::A], int64_t wa,
                                             int64_t wb, const RCriticArgs &ca, int lane, const float (&h)[8][4],
                                             float (&hn)[8][4], float (&v)[4]) {
    using R = RCriticShape<P, K>;
    using C = CriticShape<P, K>;
    constexpr int NT = 8, D = C::in_dim();
    const int tq = lane & 3;
    const bool tanh_act = ca.net_flags & kMappoTanh, feature_norm = ca.net_flags & kMappoFeatureNorm;
    // this lane's A-fragment entries of agent I's k-tile kt: (row g, col c0), (g + 8, c0), (g, c1), (g + 8, c1); zero
    // beyond obs_dim_I
    auto load = [&](auto ic, int kt, float (&q)[4]) {
        constexpr int I = decltype(ic)::value, OD = P::obs_dim(I);
        const float *r0 = src[I] + wa * OD, *r1 = src[I] + wb * OD;
        const int c0 = kt * 8 + tq, c1 = c0 + 4;
        q[0] = c0 < OD ? __ldg(r0 + c0) : 0.0f; q[1] = c0 < OD ? __ldg(r1 + c0) : 0.0f;
        q[2] = c1 < OD ? __ldg(r0 + c1) : 0.0f; q[3] = c1 < OD ? __ldg(r1 + c1) : 0.0f;
    };
    float mu0 = 0.0f, mu1 = 0.0f, rs0 = 1.0f, rs1 = 1.0f;
    if (feature_norm) {   // k-tile by k-tile (not unrolled: spread N=6 would hoist its 120 loads and spill)
        float s0 = 0.0f, s1 = 0.0f;
        static_for<P::A>([&](auto ic) {
            if constexpr (K < 0 || decltype(ic)::value == K) {
#pragma unroll 1
            for (int kt = 0; kt < MlpShape<P, 64>::kt1(decltype(ic)::value); ++kt) {
                float q[4];
                load(ic, kt, q);
                s0 += q[0] + q[2]; s1 += q[1] + q[3];
            }
            }
        });
        s0 += __shfl_xor_sync(0xffffffffu, s0, 1); s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
        s0 += __shfl_xor_sync(0xffffffffu, s0, 2); s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
        mu0 = s0 / static_cast<float>(D); mu1 = s1 / static_cast<float>(D);
        float v0 = 0.0f, v1 = 0.0f;
        static_for<P::A>([&](auto ic) {
            constexpr int I = decltype(ic)::value, OD = P::obs_dim(I);
            if constexpr (K < 0 || I == K) {
#pragma unroll 1
            for (int kt = 0; kt < MlpShape<P, 64>::kt1(I); ++kt) {
                float q[4];
                load(ic, kt, q);
                if (kt * 8 + tq < OD) { const float d0 = q[0] - mu0, d1 = q[1] - mu1; v0 += d0 * d0; v1 += d1 * d1; }
                if (kt * 8 + tq + 4 < OD) { const float d0 = q[2] - mu0, d1 = q[3] - mu1; v0 += d0 * d0; v1 += d1 * d1; }
            }
            }
        });
        v0 += __shfl_xor_sync(0xffffffffu, v0, 1); v1 += __shfl_xor_sync(0xffffffffu, v1, 1);
        v0 += __shfl_xor_sync(0xffffffffu, v0, 2); v1 += __shfl_xor_sync(0xffffffffu, v1, 2);
        rs0 = rsqrtf(v0 / static_cast<float>(D) + ca.ln_eps); rs1 = rsqrtf(v1 / static_cast<float>(D) + ca.ln_eps);
    }
    // ---- layer 1: sum over agents of [16 x K1_i] . W1[:, agent i's columns]^T, + b1 ----
    float c[NT][4];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
        const float2 b = *reinterpret_cast<const float2 *>(Wsm + R::b1_off + nt * 8 + 2 * tq);
        c[nt][0] = b.x; c[nt][1] = b.y; c[nt][2] = b.x; c[nt][3] = b.y;
    }
    static_for<P::A>([&](auto ic) {
        constexpr int I = decltype(ic)::value, OD = P::obs_dim(I);
        if constexpr (K < 0 || I == K) {
        const float *W1 = Wsm + C::w1_off(I);
#pragma unroll
        for (int kt = 0; kt < MlpShape<P, 64>::kt1(I); ++kt) {
            float q[4];
            load(ic, kt, q);
            if (feature_norm) {   // padded columns stay zero
                if (kt * 8 + tq < OD) { q[0] = (q[0] - mu0) * rs0; q[1] = (q[1] - mu1) * rs1; }
                if (kt * 8 + tq + 4 < OD) { q[2] = (q[2] - mu0) * rs0; q[3] = (q[3] - mu1) * rs1; }
            }
            const uint32_t a[4] = {to_tf32(q[0]), to_tf32(q[1]), to_tf32(q[2]), to_tf32(q[3])};
#pragma unroll
            for (int nt = 0; nt < NT; ++nt)
                mma_tf32(c[nt], a, *reinterpret_cast<const float2 *>(W1 + ((kt * NT + nt) * 32 + lane) * 2));
        }
        }
    });
    // ---- layer 2 and the base's last LayerNorm -> x ----
    uint32_t x[NT][4];
    {
        uint32_t xa[NT][4];
        act_norm_tf32_frags<NT>(xa, c, tanh_act, ca.ln_eps);
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            const float2 bb = *reinterpret_cast<const float2 *>(Wsm + R::b2_off + nt * 8 + 2 * tq);
            c[nt][0] = bb.x; c[nt][1] = bb.y; c[nt][2] = bb.x; c[nt][3] = bb.y;
#pragma unroll
            for (int kt = 0; kt < NT; ++kt)
                mma_tf32(c[nt], xa[kt], *reinterpret_cast<const float2 *>(Wsm + R::w2_off + ((kt * NT + nt) * 32 + lane) * 2));
        }
        act_norm_tf32_frags<NT>(x, c, tanh_act, ca.ln_eps);
    }
    // ---- h' = GRU(x, h), h as W_hh's A operand in TF32 (the accumulator layout is relu_tf32_frag's A layout) ----
    uint32_t ht[NT][4];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
        ht[nt][0] = to_tf32(h[nt][0]); ht[nt][1] = to_tf32(h[nt][2]);
        ht[nt][2] = to_tf32(h[nt][1]); ht[nt][3] = to_tf32(h[nt][3]);
    }
    gru_cell(Wsm + R::wih_off, Wsm + R::whh_off, Wsm + R::bih_off, Wsm + R::bhh_off, x, ht, lane, hn,
             [&](int j, float (&hf)[4]) { hf[0] = h[j][0]; hf[1] = h[j][1]; hf[2] = h[j][2]; hf[3] = h[j][3]; });
    // ---- V = W3 LN(h') + b3 ----
    uint32_t xh[NT][4];
    norm_tf32_frags<NT>(xh, hn, ca.ln_eps);
    const float2 b3 = *reinterpret_cast<const float2 *>(Wsm + R::b3_off + 2 * tq);
    v[0] = b3.x; v[1] = b3.y; v[2] = b3.x; v[3] = b3.y;
#pragma unroll
    for (int kt = 0; kt < NT; ++kt) mma_tf32(v, xh[kt], *reinterpret_cast<const float2 *>(Wsm + R::w3_off + (kt * 32 + lane) * 2));
}

// the warp's values into rec [A][n] (one row of values or final_values): the shared value for every agent
template <class P>
__device__ __forceinline__ void rcritic_store(float *rec, int64_t n, int64_t w0, int lane, int rows, const float (&v)[4]) {
    const int ra = lane >> 2, rb = ra + 8;
    if ((lane & 3) != 0) return;
#pragma unroll
    for (int s = 0; s < P::A; ++s) {
        if (ra < rows) rec[s * n + w0 + ra] = v[0];
        if (rb < rows) rec[s * n + w0 + rb] = v[2];
    }
}

// the warp's values into one agent's row rec [n] (column 0 of rows g and g + 8 in elements 0 and 2 of the quad's first
// lane)
__device__ __forceinline__ void rcritic_store_one(float *rec, int64_t w0, int lane, int rows, const float (&v)[4]) {
    const int ra = lane >> 2, rb = ra + 8;
    if ((lane & 3) != 0) return;
    if (ra < rows) rec[w0 + ra] = v[0];
    if (rb < rows) rec[w0 + rb] = v[2];
}

}  // namespace mpe
