// mpe_critic_gru.cu -- rMAPPO's recurrent centralized critic (RCriticArgs, RCriticShape in mpe_kernels.cu): one kernel
// per program of GruBuilt, compiled as a translation unit of its own so that the build runs it alongside the rest of
// the library.
#define MPE_KERNEL_TEMPLATES_ONLY
#include "mpe_kernels.cu"
#include "mpe_critic_gru.cuh"

namespace mpe {

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
