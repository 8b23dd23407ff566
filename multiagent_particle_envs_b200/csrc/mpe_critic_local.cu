// mpe_critic_local.cu -- IPPO's local critics (MAPPO with use_centralized_V = False: agent k's critic reads obs_k
// alone), compiled as a translation unit of their own so that the build runs them alongside the rest of the library:
//  - MAPPO's actor with the MLP local critics (LocalCriticShape in mpe_kernels.cu) in one launch,
//    mpe_policy_mappo_local_critic[_episode]_kernel, for the programs of local_critic_built;
//  - rIPPO's recurrent local critic after the recurrent actor's rollout, mpe_critic_gru_local_kernel, for the programs
//    of GruBuilt.
#define MPE_KERNEL_TEMPLATES_ONLY
#include "mpe_kernels.cu"
#include "mpe_critic_gru.cuh"

namespace mpe {

template <class P>
__global__ void __launch_bounds__(local_critic_block_warps<P, false>() * 32)
    mpe_policy_mappo_local_critic_kernel(const __grid_constant__ MlpCriticArgs ca) {
    mlp_rollout<P, 64, false, true, true, false, true, false, true>(ca.m.c.p, nullptr, &ca.m.c.c, ca.m.eps,
                                                                    ca.m.net_flags, nullptr, &ca.v);
}

template <class P>
__global__ void __launch_bounds__(local_critic_block_warps<P, true>() * 32)
    mpe_policy_mappo_local_critic_episode_kernel(const __grid_constant__ MlpCriticEpisodeArgs ca) {
    mlp_rollout<P, 64, true, true, true, false, true, false, true>(ca.m.c.e.p, &ca.m.c.e, &ca.m.c.c, ca.m.eps,
                                                                   ca.m.net_flags, nullptr, &ca.v);
}

template <class P>
const void *local_critic_kernel(int episodes) {
    static_assert(local_critic_built<P>(), "a program with local critics");
    return episodes ? reinterpret_cast<const void *>(mpe_policy_mappo_local_critic_episode_kernel<P>)
                    : reinterpret_cast<const void *>(mpe_policy_mappo_local_critic_kernel<P>);
}

// the programs of local_critic_built: every MAPPO program but tag 4+2 and 6+2, whose adversaries and good agents
// observe differently and whose per-agent critics do not fit next to the actor.  Where the agents observe alike
// (simple, spread N = 2..6, reference) one shared critic fits everywhere, per-agent ones on all but spread N = 5 and 6.
static_assert(!local_critic_built<Tag<4, 2, 2>>() && !local_critic_built<Tag<6, 2, 3>>() &&
              local_critic_smem_warps<Spread<4>>(4) == 7 && local_critic_smem_warps<Spread<6>>(1) == 4,
              "the programs below: tag 4+2 lacks 17 warps' room, spread N=4's four critics leave 7 warps");
template const void *local_critic_kernel<Simple<1, 1>>(int);
template const void *local_critic_kernel<Spread<2>>(int);
template const void *local_critic_kernel<Spread<3>>(int);
template const void *local_critic_kernel<Spread<4>>(int);
template const void *local_critic_kernel<Spread<5>>(int);
template const void *local_critic_kernel<Spread<6>>(int);
template const void *local_critic_kernel<Tag<3, 1, 2>>(int);
template const void *local_critic_kernel<Tag<1, 1, 2>>(int);
template const void *local_critic_kernel<Tag<2, 1, 2>>(int);
template const void *local_critic_kernel<Adversary<1, 2, 2>>(int);
template const void *local_critic_kernel<Adversary<1, 3, 3>>(int);
template const void *local_critic_kernel<Push<1, 1, 2>>(int);
template const void *local_critic_kernel<SpeakerListener>(int);
template const void *local_critic_kernel<Reference>(int);
template const void *local_critic_kernel<Crypto>(int);

// rIPPO's recurrent local critic (RCriticArgs): one weight set shared by every agent (share_policy), W1 over one
// agent's k-tiles (RCriticShape<P, 0>: every agent observes alike on these programs).  Block (x, k) stages it once and
// scans its warps' worlds as mpe_critic_gru_kernel does (rcritic_eval on agent k's records alone), with agent k's state
// (slice k of h [A][n][64] and h_rec [T][A][n][64]) and agent k's row of the values.  The scan is written out again,
// as mpe_critic_gru_separated_kernel's is, so that the existing recurrent critics keep their SASS.
template <class P>
__global__ void __launch_bounds__(kRCriticWarps * 32) mpe_critic_gru_local_kernel(const __grid_constant__ RCriticArgs ca) {
    using R = RCriticShape<P, 0>;
    constexpr int A = P::A, NT = 8;
    static_assert(LocalCriticShape<P>::shared_ok(), "one shared local critic: every agent observes alike");
    extern __shared__ __align__(16) float smem[];
    const int k = blockIdx.y;
    stage_critic_w1<P, 0, 0>(smem, ca.w1);
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
    constexpr int OD = P::obs_dim(0);
    float *const hk = ca.h + static_cast<int64_t>(k) * n * 64;               // agent k's state
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
    const float *src[A] = {};   // rcritic_eval<P, 0> reads src[0] only: agent k's records
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
        src[0] = ca.obs[k] + static_cast<int64_t>(t) * n * OD;
        rcritic_eval<P, 0>(smem, src, wa, wb, ca, lane, h, hn, v);
        rcritic_store_one(values + static_cast<int64_t>(t) * A * n, w0, lane, rows, v);
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) h[nt][e] = hn[nt][e];
        if (episodes && (t + 1) % L == 0) {   // the episode's bootstrap value, from its final observation
            const int e = t / L;
            src[0] = ca.final_obs[k] + static_cast<int64_t>(e) * n * OD;
            rcritic_eval<P, 0>(smem, src, wa, wb, ca, lane, h, hn, v);
            rcritic_store_one(final_values + static_cast<int64_t>(e) * A * n, w0, lane, rows, v);
        }
    }
    if (!episodes) {                    // the bootstrap value after the last step
        src[0] = ca.final_obs[k];
        rcritic_eval<P, 0>(smem, src, wa, wb, ca, lane, h, hn, v);
        rcritic_store_one(final_values, w0, lane, rows, v);
    }
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {   // the state after the last step, what the next call continues from
        if (ra < rows) *reinterpret_cast<float2 *>(hk + wa * 64 + nt * 8 + 2 * tq) = make_float2(h[nt][0], h[nt][1]);
        if (rb < rows) *reinterpret_cast<float2 *>(hk + wb * 64 + nt * 8 + 2 * tq) = make_float2(h[nt][2], h[nt][3]);
    }
}

template <class P>
const void *critic_gru_local_kernel() {
    static_assert(GruBuilt<P>::value, "a program with the recurrent actor");
    return reinterpret_cast<const void *>(mpe_critic_gru_local_kernel<P>);
}

// the programs of GruBuilt
template const void *critic_gru_local_kernel<Simple<1, 1>>();
template const void *critic_gru_local_kernel<Spread<2>>();
template const void *critic_gru_local_kernel<Spread<3>>();
template const void *critic_gru_local_kernel<Spread<4>>();
template const void *critic_gru_local_kernel<Spread<5>>();
template const void *critic_gru_local_kernel<Spread<6>>();
template const void *critic_gru_local_kernel<Reference>();

}  // namespace mpe
