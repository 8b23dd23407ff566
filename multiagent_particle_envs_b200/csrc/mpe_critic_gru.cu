// mpe_critic_gru.cu -- rMAPPO's recurrent centralized critic (RCriticArgs, RCriticShape in mpe_kernels.cu): one kernel
// per program of GruBuilt, compiled as a translation unit of its own so that the build runs it alongside the rest of
// the library.
#define MPE_KERNEL_TEMPLATES_ONLY
#include "mpe_kernels.cu"

namespace mpe {

// One evaluation of the critic for the warp's m-tile (rows g and g + 8 of this lane are worlds wa and wb): x =
// base(share_obs), h' = GRU(x, h) into hn, and V(LN(h')) into v (column 0 of rows g and g + 8 in elements 0 and 2 of
// the quad's first lane).  src[i] points at agent i's [n][obs_dim_i] observations of the step.  The input LayerNorm's
// fp32 two-pass statistics over all D entries come from the A fragments themselves (a row's entries are spread over
// the 4 lanes of a quad); the records are then read a third time, normalised, rounded to TF32 and multiplied by agent
// i's k-tiles of W1.  Layers 2 and 3 are MAPPO's (act_norm_tf32_frags), the cell the recurrent actor's (gru_cell).
template <class P>
__device__ __forceinline__ void rcritic_eval(const float *__restrict__ Wsm, const float *const (&src)[P::A], int64_t wa,
                                             int64_t wb, const RCriticArgs &ca, int lane, const float (&h)[8][4],
                                             float (&hn)[8][4], float (&v)[4]) {
    using R = RCriticShape<P>;
    using C = CriticShape<P>;
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
#pragma unroll 1
            for (int kt = 0; kt < MlpShape<P, 64>::kt1(decltype(ic)::value); ++kt) {
                float q[4];
                load(ic, kt, q);
                s0 += q[0] + q[2]; s1 += q[1] + q[3];
            }
        });
        s0 += __shfl_xor_sync(0xffffffffu, s0, 1); s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
        s0 += __shfl_xor_sync(0xffffffffu, s0, 2); s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
        mu0 = s0 / static_cast<float>(D); mu1 = s1 / static_cast<float>(D);
        float v0 = 0.0f, v1 = 0.0f;
        static_for<P::A>([&](auto ic) {
            constexpr int I = decltype(ic)::value, OD = P::obs_dim(I);
#pragma unroll 1
            for (int kt = 0; kt < MlpShape<P, 64>::kt1(I); ++kt) {
                float q[4];
                load(ic, kt, q);
                if (kt * 8 + tq < OD) { const float d0 = q[0] - mu0, d1 = q[1] - mu1; v0 += d0 * d0; v1 += d1 * d1; }
                if (kt * 8 + tq + 4 < OD) { const float d0 = q[2] - mu0, d1 = q[3] - mu1; v0 += d0 * d0; v1 += d1 * d1; }
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

// Each warp scans its 16 worlds over t = 0 .. T - 1 with h in registers; one block per SM stages the weights once.
template <class P>
__global__ void __launch_bounds__(kRCriticWarps * 32) mpe_critic_gru_kernel(const __grid_constant__ RCriticArgs ca) {
    using R = RCriticShape<P>;
    using C = CriticShape<P>;
    constexpr int A = P::A, NT = 8;
    extern __shared__ __align__(16) float smem[];
    static_for<A>([&](auto ic) {
        constexpr int i = decltype(ic)::value;
        stage_critic_w1<P, i>(smem + C::w1_off(i), ca.w1);
    });
    stage_fragments<NT, NT, true>(smem + R::w2_off, ca.w2, 64, 64);
    stage_fragments<NT, R::NG, true>(smem + R::wih_off, ca.w_ih, 192, 64);
    stage_fragments<NT, R::NG, true>(smem + R::whh_off, ca.w_hh, 192, 64);
    stage_fragments<NT, 1, true>(smem + R::w3_off, ca.w3, 1, 64);
    for (int q = threadIdx.x; q < 64; q += blockDim.x) {
        smem[R::b1_off + q] = ca.b1[q];
        smem[R::b2_off + q] = ca.b2[q];
    }
    for (int q = threadIdx.x; q < 192; q += blockDim.x) {
        smem[R::bih_off + q] = ca.b_ih[q];
        smem[R::bhh_off + q] = ca.b_hh[q];
    }
    for (int q = threadIdx.x; q < 8; q += blockDim.x) smem[R::b3_off + q] = q == 0 ? ca.b3[0] : 0.0f;
    __syncthreads();

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t n = ca.n;
    const int64_t w0 = (static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + warp) * 16;
    if (w0 >= n) return;
    const int rows = (n - w0) < 16 ? static_cast<int>(n - w0) : 16;
    // this lane's rows g and g + 8 in the accumulator layout (units nt * 8 + 2 tq, + 1); idle rows replay world w0 and
    // store nothing
    const int tq = lane & 3, ra = lane >> 2, rb = ra + 8;
    const int64_t wa = w0 + (ra < rows ? ra : 0), wb = w0 + (rb < rows ? rb : 0);
    const bool episodes = ca.L > 0;
    const int L = episodes ? ca.L : ca.T;
    float h[NT][4];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
        const float2 va = episodes ? make_float2(0.0f, 0.0f) : *reinterpret_cast<const float2 *>(ca.h + wa * 64 + nt * 8 + 2 * tq);
        const float2 vb = episodes ? make_float2(0.0f, 0.0f) : *reinterpret_cast<const float2 *>(ca.h + wb * 64 + nt * 8 + 2 * tq);
        h[nt][0] = va.x; h[nt][1] = va.y; h[nt][2] = vb.x; h[nt][3] = vb.y;
    }
    const float *src[A];
    float hn[NT][4], v[4];
#pragma unroll 1
    for (int t = 0; t < ca.T; ++t) {
        if (episodes && t % L == 0) {   // every episode starts from h = 0 (MAPPO's mask after done)
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) h[nt][0] = h[nt][1] = h[nt][2] = h[nt][3] = 0.0f;
        }
        if (ca.h_rec != nullptr) {      // the h this step's critic consumes
            float *qa = ca.h_rec + (static_cast<int64_t>(t) * n + wa) * 64 + 2 * tq;
            float *qb = ca.h_rec + (static_cast<int64_t>(t) * n + wb) * 64 + 2 * tq;
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) {
                if (ra < rows) *reinterpret_cast<float2 *>(qa + nt * 8) = make_float2(h[nt][0], h[nt][1]);
                if (rb < rows) *reinterpret_cast<float2 *>(qb + nt * 8) = make_float2(h[nt][2], h[nt][3]);
            }
        }
        static_for<A>([&](auto ic) {
            constexpr int i = decltype(ic)::value;
            src[i] = ca.obs[i] + static_cast<int64_t>(t) * n * P::obs_dim(i);
        });
        rcritic_eval<P>(smem, src, wa, wb, ca, lane, h, hn, v);
        rcritic_store<P>(ca.values + static_cast<int64_t>(t) * A * n, n, w0, lane, rows, v);
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) h[nt][e] = hn[nt][e];
        if (episodes && (t + 1) % L == 0) {   // the episode's bootstrap value, from its final observation
            const int e = t / L;
            static_for<A>([&](auto ic) {
                constexpr int i = decltype(ic)::value;
                src[i] = ca.final_obs[i] + static_cast<int64_t>(e) * n * P::obs_dim(i);
            });
            rcritic_eval<P>(smem, src, wa, wb, ca, lane, h, hn, v);
            rcritic_store<P>(ca.final_values + static_cast<int64_t>(e) * A * n, n, w0, lane, rows, v);
        }
    }
    if (!episodes) {                    // the bootstrap value after the last step
        static_for<A>([&](auto ic) {
            constexpr int i = decltype(ic)::value;
            src[i] = ca.final_obs[i];
        });
        rcritic_eval<P>(smem, src, wa, wb, ca, lane, h, hn, v);
        rcritic_store<P>(ca.final_values, n, w0, lane, rows, v);
    }
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {   // the state after the last step, what the next call continues from
        if (ra < rows) *reinterpret_cast<float2 *>(ca.h + wa * 64 + nt * 8 + 2 * tq) = make_float2(h[nt][0], h[nt][1]);
        if (rb < rows) *reinterpret_cast<float2 *>(ca.h + wb * 64 + nt * 8 + 2 * tq) = make_float2(h[nt][2], h[nt][3]);
    }
}

template <class P>
const void *critic_gru_kernel() {
    static_assert(GruBuilt<P>::value, "a program with the recurrent actor");
    return reinterpret_cast<const void *>(mpe_critic_gru_kernel<P>);
}

// the programs of GruBuilt
template const void *critic_gru_kernel<Simple<1, 1>>();
template const void *critic_gru_kernel<Spread<2>>();
template const void *critic_gru_kernel<Spread<3>>();
template const void *critic_gru_kernel<Spread<4>>();
template const void *critic_gru_kernel<Spread<5>>();
template const void *critic_gru_kernel<Spread<6>>();
template const void *critic_gru_kernel<Reference>();

}  // namespace mpe
