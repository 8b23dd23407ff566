// mpe_gru_separated.cu -- rMAPPO's separated runner for the programs of GruSeparatedBuilt: every agent's recurrent actor
// (mpe_gru_image_kernel, mpe_policy_gru_separated[_episode]_kernel, see mpe_kernels.cu) and every agent's recurrent
// critic (mpe_critic_gru_separated_kernel), compiled as a translation unit of their own so that the build runs them
// alongside the rest of the library.
#define MPE_KERNEL_TEMPLATES_ONLY
#include "mpe_kernels.cu"
#include "mpe_critic_gru.cuh"

namespace mpe {

// rMAPPO's per-agent recurrent critics (RCriticSeparatedArgs): block (x, k) stages critic k's weights once and scans
// its warps' worlds as mpe_critic_gru_kernel does (rcritic_eval), with critic k's state (slice k of h and h_rec) and only
// agent k's row of the values.  The critics do not affect the trajectory, so they run after the rollout over its
// observation records and need no restaging.  The scan is mpe_critic_gru_kernel's written out again: sharing it through
// a template changed the shared critic's SASS and registers.
template <class P>
__global__ void __launch_bounds__(kRCriticWarps * 32)
    mpe_critic_gru_separated_kernel(const __grid_constant__ RCriticSeparatedArgs sa) {
    using R = RCriticShape<P>;
    using C = CriticShape<P>;
    constexpr int A = P::A, NT = 8;
    extern __shared__ __align__(16) float smem[];
    const RCriticArgs &ca = sa.c;
    const int k = blockIdx.y;
    static_for<A>([&](auto ic) {
        constexpr int i = decltype(ic)::value;
        stage_critic_w1<P, i>(smem + C::w1_off(i), sa.w[0][k]);
    });
    stage_fragments<NT, NT, true>(smem + R::w2_off, sa.w[2][k], 64, 64);
    stage_fragments<NT, R::NG, true>(smem + R::wih_off, sa.w[4][k], 192, 64);
    stage_fragments<NT, R::NG, true>(smem + R::whh_off, sa.w[6][k], 192, 64);
    stage_fragments<NT, 1, true>(smem + R::w3_off, sa.w[8][k], 1, 64);
    for (int q = threadIdx.x; q < 64; q += blockDim.x) {
        smem[R::b1_off + q] = sa.w[1][k][q];
        smem[R::b2_off + q] = sa.w[3][k][q];
    }
    for (int q = threadIdx.x; q < 192; q += blockDim.x) {
        smem[R::bih_off + q] = sa.w[5][k][q];
        smem[R::bhh_off + q] = sa.w[7][k][q];
    }
    for (int q = threadIdx.x; q < 8; q += blockDim.x) smem[R::b3_off + q] = q == 0 ? sa.w[9][k][0] : 0.0f;
    __syncthreads();

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t n = ca.n;
    float *const hk = ca.h + static_cast<int64_t>(k) * n * 64;               // critic k's state
    float *const values = ca.values + static_cast<int64_t>(k) * n;           // agent k's row
    float *const final_values = ca.final_values + static_cast<int64_t>(k) * n;
    const int64_t w0 = (static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + warp) * 16;
    if (w0 >= n) return;
    const int rows = (n - w0) < 16 ? static_cast<int>(n - w0) : 16;
    const int tq = lane & 3, ra = lane >> 2, rb = ra + 8;
    const int64_t wa = w0 + (ra < rows ? ra : 0), wb = w0 + (rb < rows ? rb : 0);
    const bool episodes = ca.L > 0;
    const int L = episodes ? ca.L : ca.T;
    float h[NT][4];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
        const float2 va = episodes ? make_float2(0.0f, 0.0f) : *reinterpret_cast<const float2 *>(hk + wa * 64 + nt * 8 + 2 * tq);
        const float2 vb = episodes ? make_float2(0.0f, 0.0f) : *reinterpret_cast<const float2 *>(hk + wb * 64 + nt * 8 + 2 * tq);
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
        if (ca.h_rec != nullptr) {      // the h this step's critic consumes, row (t, k) of [T][A][n][64]
            float *qa = ca.h_rec + ((static_cast<int64_t>(t) * A + k) * n + wa) * 64 + 2 * tq;
            float *qb = ca.h_rec + ((static_cast<int64_t>(t) * A + k) * n + wb) * 64 + 2 * tq;
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
        rcritic_store_one(values + static_cast<int64_t>(t) * A * n, w0, lane, rows, v);
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
            rcritic_store_one(final_values + static_cast<int64_t>(e) * A * n, w0, lane, rows, v);
        }
    }
    if (!episodes) {                    // the bootstrap value after the last step
        static_for<A>([&](auto ic) {
            constexpr int i = decltype(ic)::value;
            src[i] = ca.final_obs[i];
        });
        rcritic_eval<P>(smem, src, wa, wb, ca, lane, h, hn, v);
        rcritic_store_one(final_values, w0, lane, rows, v);
    }
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {   // the state after the last step, what the next call continues from
        if (ra < rows) *reinterpret_cast<float2 *>(hk + wa * 64 + nt * 8 + 2 * tq) = make_float2(h[nt][0], h[nt][1]);
        if (rb < rows) *reinterpret_cast<float2 *>(hk + wb * 64 + nt * 8 + 2 * tq) = make_float2(h[nt][2], h[nt][3]);
    }
}

template <class P>
const void *gru_separated_kernel(int which) {
    static_assert(GruSeparatedBuilt<P>::value && MlpBuilt<P>::value, "a program with per-agent recurrent actors");
    switch (which) {
    case 0: return reinterpret_cast<const void *>(mpe_gru_image_kernel<P>);
    case 1: return reinterpret_cast<const void *>(mpe_policy_gru_separated_kernel<P>);
    case 2: return reinterpret_cast<const void *>(mpe_policy_gru_separated_episode_kernel<P>);
    default: return reinterpret_cast<const void *>(mpe_critic_gru_separated_kernel<P>);
    }
}

// the programs of GruSeparatedBuilt
template const void *gru_separated_kernel<SpeakerListener>(int);

}  // namespace mpe
