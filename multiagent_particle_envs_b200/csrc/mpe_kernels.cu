// mpe_kernels.cu -- the hot path of multiagent-particle-envs for a batch of worlds, sm_90a.
//
//   kFusedStep  MultiAgentEnv.step            environment.py:80-104   (one launch)
//   kSetAction  MultiAgentEnv._set_action     environment.py:144-192
//   kWorldStep  World.step                    core.py:117-131
//   kObserve    scenario.observation/reward + step glue (also used by reset)
//
// All four are the same kernel template with phases compiled in or out, so the fused step is
// bit-identical to set_action -> world_step -> observe.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <type_traits>
#include <utility>

#include <nvtx3/nvToolsExt.h>   // header-only NVTX v3: ranges cost a few ns unless a profiler is attached

#include "mpe_scenarios.cuh"

namespace mpe {

template <int... I, class F>
__device__ __forceinline__ void static_for_impl(std::integer_sequence<int, I...>, F &&f) {
    (f(std::integral_constant<int, I>{}), ...);
}
template <int N, class F>
__device__ __forceinline__ void static_for(F &&f) {
    static_for_impl(std::make_integer_sequence<int, N>{}, static_cast<F &&>(f));
}

template <class P>
struct Shape {
    // warp-private staging, in floats: [lead: 4][action tiles of all agents][one observation slot]
    // Every observation tile of a warp shares the slot (write rows, sync, stream out, sync).  A slot per tile would
    // make world_comm's staging 22 KB per warp and let shared memory cap residency at 10 warps per SM; shared, it is
    // 6 KB and registers are the limit (16 warps per SM).
    // The tiles start 16 bytes into the staging.  At offset 0, world_comm's fused step at 32 768 worlds measured 8-20 %
    // slower on an H100 SXM (400 W), while spread N=3, tag and the open-loop rollout measured 0.3-8 % faster.
    static constexpr int kLeadFloats = 4;
    __host__ __device__ static constexpr int act_floats(int i) { return 32 * (P::act_dim(i) | 1); }
    __host__ __device__ static constexpr int act_off(int i) { int s = kLeadFloats; for (int j = 0; j < i; ++j) s += act_floats(j); return s; }
    __host__ __device__ static constexpr bool act_dense(int i) { return (P::act_dim(i) | 1) == P::act_dim(i); }
    __host__ __device__ static constexpr bool all_act_dense() { for (int i = 0; i < P::A; ++i) if (!act_dense(i)) return false; return true; }
    __host__ __device__ static constexpr int obs_pitch(int i) {
        const int od = P::obs_dim(i), unit = (od % 2 == 0) ? 2 : 1;
        return ((od / unit) | 1) * unit;
    }
    __host__ __device__ static constexpr int obs_floats(int i) { return (32 * obs_pitch(i) + 3) & ~3; }
    __host__ __device__ static constexpr int obs_base() { return act_off(P::A); }
    __host__ __device__ static constexpr int warp_floats() {
        int m = 0;
        for (int i = 0; i < P::A; ++i) m = obs_floats(i) > m ? obs_floats(i) : m;
        return (obs_base() + m + 3) & ~3;
    }
    // cp.async destinations and the LDS.128 of the tile streams need every tile on a 16-byte boundary
    __host__ __device__ static constexpr bool tiles_aligned() { for (int i = 0; i <= P::A; ++i) if (act_off(i) % 4) return false; return true; }
    static_assert(tiles_aligned(), "every staging tile starts at a multiple of 4 floats");
    static constexpr int kWarpFloats = warp_floats();
    static constexpr int kWarpBytes = kWarpFloats * 4;
    // K-step rollout: a second set of action tiles behind the regular staging (step t+1 is prefetched while step t runs)
    static constexpr int kRolloutWarpFloats = kWarpFloats + ((obs_base() + 3) & ~3);
    static constexpr int kRolloutWarpBytes = kRolloutWarpFloats * 4;
    static constexpr int kNC = P::NS * P::DIMC;
};

// World.step physics for one world held in registers (core.py:134-169)
template <class P>
__device__ __forceinline__ void physics(const DevDesc &d, typename P::W &w, const float (&ux)[P::A],
                                        const float (&uy)[P::A]) {
    constexpr int A = P::A, L = P::L;
    float2 F[A];   // (x, y) force pairs
#pragma unroll
    for (int i = 0; i < A; ++i) F[i] = make_float2(ux[i], uy[i]);  // apply_action_force (core.py:134-140)
    const float k = d.contact_margin, cf = d.contact_force;
    // apply_environment_force (core.py:143-155): pairs (a, b), a < b, agents then landmarks.
    // Landmark-landmark pairs move nothing and are dropped at compile time.
#pragma unroll
    for (int a = 0; a < A; ++a) {
#pragma unroll
        for (int b = a + 1; b < A + L; ++b) {
            const bool b_agent = b < A;
            const int bi = b_agent ? b : 0, bl = b_agent ? 0 : b - A;
            // get_collision_force (core.py:181-182): the collide flags are structural constants of the
            // scenario program, so non-colliding pairs vanish at compile time and the remaining pairs form
            // one straight-line block that the scheduler interleaves freely
            if (!(P::agent_collides(a) && (b_agent ? P::agent_collides(bi) : P::landmark_collides(bl)))) continue;
            const float bx = b_agent ? w.px[bi] : w.lx[bl];
            const float by = b_agent ? w.py[bi] : w.ly[bl];
            const float sb = b_agent ? d.a_size[bi] : d.l_size[bl];
            const float2 dl = sub2(make_float2(w.px[a], w.py[a]), make_float2(bx, by));
            const float2 f = pair_force(dl.x, dl.y, __fadd_rn(d.a_size[a], sb), cf, k, d.inv_margin);   // :186-193
            if (P::movable(a)) F[a] = add2(F[a], f);                        // :194, 149-151
            if (b_agent && P::movable(bi)) F[bi] = sub2(F[bi], f);          // :195, 152-154
        }
    }
    // integrate_state (core.py:158-169)
#pragma unroll
    for (int i = 0; i < A; ++i) {
        if (!P::movable(i)) continue;
        const float4 r = integrate_entity<P::kSpeedLimit>(w.px[i], w.py[i], w.vx[i], w.vy[i], F[i].x, F[i].y, d.keep,
                                                          d.a_dt_over_mass[i], d.dt, d.a_max_speed[i]);
        w.px[i] = r.x; w.py[i] = r.y; w.vx[i] = r.z; w.vy[i] = r.w;
    }
}


// _set_action's movement force (environment.py:173-181) from the movement probabilities p1..p4.  The force starts at
// +0: 0 + (-0) is +0, so the addition is part of the result's bits.  sens is taken by reference so that it is read
// after the additions, the order the callers' instruction schedules were tuned with.
__device__ __forceinline__ float2 movement_force(float p1, float p2, float p3, float p4, const float &sens) {
    float x = 0.0f, y = 0.0f;                                           // :145
    x += p1 - p2;                                                       // :174
    y += p3 - p4;                                                       // :175
    // explicit multiplies: must not be contracted into the force accumulation, or the fused
    // step would round differently from set_action -> world_step
    return make_float2(__fmul_rn(x, sens), __fmul_rn(y, sens));        // :178-181
}

// MultiAgentEnv._set_action (environment.py:144-192) for this lane's world, from the warp's staged action tiles
// (s_act = the warp's staging base; tile i starts at Shape<P>::act_off(i))
template <class P, bool ALLOW_FORCE_DISCRETE = true>
__device__ __forceinline__ void decode_rows(const float *s_act, int lane, const DevDesc &d, uint32_t flags,
                                            float (&ux)[P::A], float (&uy)[P::A], float *cact) {
    static_for<P::A>([&](auto ic) {
        constexpr int i = decltype(ic)::value;
        constexpr int AD = P::act_dim(i);
        constexpr int OFF = Shape<P>::act_off(i);
        const float *row = s_act + OFF + lane * Tile<AD>::kStride;
        int off = 0;
        float2 u = make_float2(0.0f, 0.0f);                             // immovable: no force
        if constexpr (P::movable(i)) {
            float p0 = row[0], p1 = row[1], p2 = row[2], p3 = row[3], p4 = row[4];
            if (ALLOW_FORCE_DISCRETE && (flags & MPE_FLAG_FORCE_DISCRETE_ACTION)) {   // :169-172 (first arg-max)
                int best = 0;
                float bv = p0;
                if (p1 > bv) { bv = p1; best = 1; }
                if (p2 > bv) { bv = p2; best = 2; }
                if (p3 > bv) { bv = p3; best = 3; }
                if (p4 > bv) { bv = p4; best = 4; }
                p1 = best == 1 ? 1.0f : 0.0f; p2 = best == 2 ? 1.0f : 0.0f;
                p3 = best == 3 ? 1.0f : 0.0f; p4 = best == 4 ? 1.0f : 0.0f;
            }
            u = movement_force(p1, p2, p3, p4, d.a_sens[i]);
            off = 5;
        }
        ux[i] = u.x;
        uy[i] = u.y;
        if constexpr (i < P::NS) {                                      // :183-190 speakers come first
#pragma unroll
            for (int q = 0; q < P::DIMC; ++q) cact[i * P::DIMC + q] = row[off + q];
        }
    });
}

// The warp's tile in a persistent rollout: worlds [w0, w0 + rows) of the launch's range [begin, end), one per lane.
// Lanes past the range (in the batch's last, partial tile) are inactive: they shadow world w0 and never store.  n is the
// kernel's copy of StepArgs::n, read at entry: a read of a.n after memory-clobbering inline asm (cp.async)
// would be a second load.
struct WarpTile {
    int lane, rows;
    bool active;
    int64_t n, w0, wi;
};
__device__ __forceinline__ WarpTile warp_tile(int lane, int64_t n, int64_t w0, int64_t end) {
    const int rows = (end - w0) < 32 ? static_cast<int>(end - w0) : 32;
    const bool active = lane < rows;
    return {lane, rows, active, n, w0, w0 + (active ? lane : 0)};
}

// this lane's world from HBM into registers: positions and velocities, landmarks, the utterances, the goals
template <class P>
__device__ __forceinline__ void load_world(const StepArgs &a, const WarpTile &wt, typename P::W &w) {
    const int64_t n = wt.n, wi = wt.wi;
#pragma unroll
    for (int i = 0; i < P::A; ++i) {
        const float4 v = a.pv[i * n + wi];
        w.px[i] = v.x; w.py[i] = v.y; w.vx[i] = v.z; w.vy[i] = v.w;
    }
#pragma unroll
    for (int l = 0; l < P::L; ++l) {
        const float2 v = a.lm[l * n + wi];
        w.lx[l] = v.x; w.ly[l] = v.y;
    }
#pragma unroll
    for (int q = 0; q < Shape<P>::kNC; ++q) w.c[q] = a.comm[q * n + wi];
#pragma unroll
    for (int q = 0; q < P::G; ++q) w.g[q] = a.goal[q * n + wi];
}

// the state a rollout changes back to HBM (active lanes only): the movable agents' positions and velocities (every
// agent's with ALL_AGENTS, after a reset has moved the immovable ones too), then the utterances
template <class P, bool ALL_AGENTS = false>
__device__ __forceinline__ void store_world(const StepArgs &a, const typename P::W &w, const WarpTile &wt) {
    const int64_t n = wt.n, wi = wt.wi;
#pragma unroll
    for (int i = 0; i < P::A; ++i)
        if (ALL_AGENTS || P::movable(i)) a.pv[i * n + wi] = make_float4(w.px[i], w.py[i], w.vx[i], w.vy[i]);
#pragma unroll
    for (int q = 0; q < Shape<P>::kNC; ++q) a.comm[q * n + wi] = w.c[q];
}

// one rollout step's rewards (scenario.reward, summed over the agents with MPE_FLAG_SHARED_REWARD as the fused step
// does), added to the running returns in step order and written to the optional record ra.rew_steps[tg][A][n]
template <class P, class Args>
__device__ __forceinline__ void rollout_rewards(const Args &ra, const typename P::W &w, float (&rsum)[P::A], int tg,
                                                const WarpTile &wt) {
    float rew[P::A];
    P::reward(ra.s.d, w, rew, nullptr);
    if (ra.s.flags & MPE_FLAG_SHARED_REWARD) {
        float sum = 0.0f;
#pragma unroll
        for (int i = 0; i < P::A; ++i) sum += rew[i];
#pragma unroll
        for (int i = 0; i < P::A; ++i) rew[i] = sum;
    }
#pragma unroll
    for (int i = 0; i < P::A; ++i) rsum[i] = __fadd_rn(rsum[i], rew[i]);
    if (ra.rew_steps != nullptr && wt.active) {
#pragma unroll
        for (int i = 0; i < P::A; ++i) ra.rew_steps[(static_cast<int64_t>(tg) * P::A + i) * wt.n + wt.wi] = rew[i];
    }
}

// one agent's observation rows of the warp's tile, staged in shared memory at `tile` (ObsTile<OD> pitch), to g: as
// coalesced 16-byte stores (LDS.128 -> STG.128) if the tile is whole and g aligned, else row by row
template <int OD>
__device__ __forceinline__ void store_obs_rows(float *g, const float *tile, int lane, int rows, bool active) {
    if (rows == 32 && (reinterpret_cast<uintptr_t>(g) & 15u) == 0) {
        obs_tile_store<OD>(g, tile, lane);
    } else if (active) {
#pragma unroll
        for (int k = 0; k < OD; ++k) g[lane * OD + k] = tile[lane * ObsTile<OD>::kPitch + k];
    }
}

// observation rows of one 32-world tile: full warps write each agent's rows into the warp's observation slot and
// stream them out as coalesced 16-byte stores (not a TMA bulk store: the warp would have to stay resident until the
// copy engine has read its shared memory); the batch's last, partial warp writes its rows straight to global memory.
template <class P>
__device__ __forceinline__ void write_observations(const StepArgs &a, const DevDesc &d, const typename P::W &w, float *slot,
                                                   int lane, int rows, bool active, int64_t w0, int64_t wi) {
    constexpr int A = P::A;
    if (rows == 32) {
        static_for<A>([&](auto ic) {
            constexpr int i = decltype(ic)::value;
            constexpr int OD = P::obs_dim(i);
            TileWriter<OD> o(slot, lane);
            P::template observe<i>(d, w, o);
            __syncwarp();
            obs_tile_store<OD>(a.obs[i] + w0 * OD, slot, lane);
            __syncwarp();
        });
    } else if (active) {  // the batch's last, partial warp: rows go straight to global memory
        static_for<A>([&](auto ic) {
            constexpr int i = decltype(ic)::value;
            RowWriter o{a.obs[i] + wi * P::obs_dim(i)};
            P::template observe<i>(d, w, o);
        });
    }
}

// the end of a rollout: the final state's observations (through the observation slot), then the returns rsum (RETURNS:
// the episode forms write theirs per episode) and done = 0 (done_callback is None, environment.py:132-135)
template <class P, bool RETURNS = true>
__device__ __forceinline__ void finish_rollout(const StepArgs &a, typename P::W &w, float *slot, const WarpTile &wt,
                                               const float (&rsum)[P::A]) {
    P::prepare(a.d, w);
    write_observations<P>(a, a.d, w, slot, wt.lane, wt.rows, wt.active, wt.w0, wt.wi);
    if (wt.active) {
#pragma unroll
        for (int i = 0; i < P::A; ++i) {
            if constexpr (RETURNS) a.rew[i * wt.n + wt.wi] = rsum[i];
            a.done[i * wt.n + wt.wi] = 0;
        }
    }
}

// __launch_bounds__(kMaxThreads, 1): 512 threads x 1 block = a 128-register budget.
//
// HOT (fused step only): the specialisation the launcher uses whenever it can -- whole 32-world tiles, 16-byte aligned
// action rows, float action vectors without force_discrete_action, cp.async staging.  It contains none of the cold
// alternatives (partial-tile scalar paths, integer decode, arg-max), i.e. about half the static code of
// the general kernel: with few resident warps per scheduler the step is bound by each warp's own instruction stream,
// including instruction-fetch stalls across the skipped cold blocks.  Same arithmetic, same order: bit-identical.
// A ragged tail and every other flag combination run on the general kernel.
//
// DENSE (HOT only): the same code compiled for an 80-register budget (__launch_bounds__(128, 6): 24 instead of 16
// resident warps per SM).  Only instantiated for programs that fit 80 registers without spilling (P::kLowRegVariant:
// the tag family up to 6 agents, spread N=4) and only launched when the batch has more tiles than the 128-register
// kernel keeps resident (> #SMs x 16 warps): there occupancy matters more, below it the register-rich version is
// preferred.
template <class P, int MODE, bool HOT = false, bool DENSE = false>
__global__ void __launch_bounds__(DENSE ? 128 : kMaxThreads, DENSE ? 6 : 1) mpe_kernel(const __grid_constant__ StepArgs a) {
    static_assert(!DENSE || HOT, "the low-register build exists for the HOT fused step only");
    static_assert(!HOT || (MODE == kFusedStep && Shape<P>::all_act_dense()), "HOT = plain fused step, dense tiles");
    constexpr int A = P::A, L = P::L, NC = Shape<P>::kNC;
    extern __shared__ __align__(16) float smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t n = a.n;
    const int64_t end = a.begin + a.count;
    const int64_t w0 = a.begin + (static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + warp) * 32;
    // Programmatic dependent launch (MPE_B200_PDL, see launch()): the index arithmetic and the first touches of the
    // parameter block (constant-bank misses) run before the wait; no global memory is touched before the previous
    // grid has completed and flushed.  A warp that exits early counts as having released the dependent grid.
    if (a.flags & kFlagPdlEarly) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    if (w0 >= end) return;  // whole warp exits together
    const int rows = HOT ? 32 : ((end - w0) < 32 ? static_cast<int>(end - w0) : 32);
    const bool active = HOT ? true : (lane < rows);
    const int64_t wi = w0 + (active ? lane : 0);  // inactive lanes shadow row 0 and never store
    float *s_warp = smem + warp * Shape<P>::kWarpFloats;
    const DevDesc &d = a.d;
    {   // pull the parameter lines that the load phase needs into registers / the constant cache now
        uintptr_t touch = reinterpret_cast<uintptr_t>(a.pv) ^ reinterpret_cast<uintptr_t>(a.lm) ^
                          reinterpret_cast<uintptr_t>(a.obs[0]) ^ reinterpret_cast<uintptr_t>(a.rew) ^ a.flags ^
                          __float_as_uint(d.dt) ^ __float_as_uint(d.a_size[0]);
        asm volatile("" ::"l"(touch));
    }
    asm volatile("griddepcontrol.wait;" ::: "memory");

    // ---- action tiles: asynchronous copies (cp.async) issued FIRST, so that they fly together
    //      with the state loads -------------------------------------------------------------------------
    bool bulk = false;
    if constexpr (HOT) {
        static_for<A>([&](auto ic) {
            constexpr int i = decltype(ic)::value;
            constexpr int AD = P::act_dim(i), kVec = 32 * AD / 4;
            const float *g = a.act[i] + w0 * AD;
            float *sdst = s_warp + Shape<P>::act_off(i);
#pragma unroll
            for (int q0 = 0; q0 < kVec; q0 += 32)
                if (q0 + 32 <= kVec || q0 + lane < kVec) cp_async16(sdst + 4 * (q0 + lane), g + 4 * (q0 + lane));
        });
    } else if constexpr ((MODE == kFusedStep || MODE == kSetAction) && Shape<P>::all_act_dense()) {
        uintptr_t bits = 0;
#pragma unroll
        for (int i = 0; i < A; ++i) bits |= reinterpret_cast<uintptr_t>(a.act[i]);
        // warp-uniform; integer actions (discrete_action_input) are one or two words per world and need no tile
        bulk = (rows == 32) && ((bits & 15u) == 0) && !(a.flags & MPE_FLAG_DISCRETE_ACTION_INPUT);
        if (bulk) {
            // every lane copies 16-byte pieces of the (contiguous) tiles straight into shared memory
            static_for<A>([&](auto ic) {
                constexpr int i = decltype(ic)::value;
                constexpr int AD = P::act_dim(i), kVec = 32 * AD / 4;
                const float *g = a.act[i] + w0 * AD;
                float *sdst = s_warp + Shape<P>::act_off(i);
#pragma unroll
                for (int q0 = 0; q0 < kVec; q0 += 32)
                    if (q0 + 32 <= kVec || q0 + lane < kVec) cp_async16(sdst + 4 * (q0 + lane), g + 4 * (q0 + lane));
            });
        }
    }

    typename P::W w;
    // ---- state loads (issued first so they overlap the action staging) ---------------------
    if constexpr (MODE != kSetAction) {
#pragma unroll
        for (int i = 0; i < A; ++i) {
            const float4 v = a.pv[i * n + wi];
            w.px[i] = v.x; w.py[i] = v.y; w.vx[i] = v.z; w.vy[i] = v.w;
        }
#pragma unroll
        for (int l = 0; l < L; ++l) {
            const float2 v = a.lm[l * n + wi];
            w.lx[l] = v.x; w.ly[l] = v.y;
        }
        if constexpr (MODE == kObserve && NC > 0) {
#pragma unroll
            for (int q = 0; q < NC; ++q) w.c[q] = a.comm[q * n + wi];
        }
        if constexpr ((MODE == kObserve || MODE == kFusedStep) && P::G > 0) {
#pragma unroll
            for (int q = 0; q < P::G; ++q) w.g[q] = a.goal[q * n + wi];
        }
    }

    if (a.flags & kFlagPdlAfterIssue) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    float ux[A], uy[A];
    float cact[NC > 0 ? NC : 1];
    // ---- MultiAgentEnv._set_action (environment.py:144-192) --------------------------------
    if constexpr (HOT) {
        cp_async_wait_all();
        __syncwarp();
        decode_rows<P, false>(s_warp, lane, d, a.flags, ux, uy, cact);
    } else if constexpr (MODE == kFusedStep || MODE == kSetAction) {
        if (a.flags & MPE_FLAG_DISCRETE_ACTION_INPUT) {
            // env.discrete_action_input (environment.py:161-167, 185-187): act_n[i] is int32 [n_env][n_sub_i], one index
            // per sub-action (movement 0..4, then the utterance 0..dim_c-1); consecutive lanes read consecutive words
            static_for<A>([&](auto ic) {
                constexpr int i = decltype(ic)::value;
                constexpr int NSUB = (P::movable(i) ? 1 : 0) + (i < P::NS ? 1 : 0);
                const int32_t *row = reinterpret_cast<const int32_t *>(a.act[i]) + wi * NSUB;
                float x = 0.0f, y = 0.0f;                                       // :145, 162
                int off = 0;
                if constexpr (P::movable(i)) {
                    const int k = row[0];
                    x = k == 1 ? -1.0f : (k == 2 ? 1.0f : 0.0f);                // :164-165
                    y = k == 3 ? -1.0f : (k == 4 ? 1.0f : 0.0f);                // :166-167
                    x = __fmul_rn(x, d.a_sens[i]);                              // :178-181
                    y = __fmul_rn(y, d.a_sens[i]);
                    off = 1;
                }
                ux[i] = x;
                uy[i] = y;
                if constexpr (i < P::NS) {                                      // :186-187 one-hot utterance
                    const int k = row[off];
#pragma unroll
                    for (int q = 0; q < P::DIMC; ++q) cact[i * P::DIMC + q] = (k == q) ? 1.0f : 0.0f;
                }
            });
        } else {
        if (bulk) {
            cp_async_wait_all();
            __syncwarp();
        } else {
            static_for<A>([&](auto ic) {
                constexpr int i = decltype(ic)::value;
                constexpr int AD = P::act_dim(i);
                constexpr int OFF = Shape<P>::act_off(i);
                tile_load<AD>(s_warp + OFF, a.act[i] + w0 * AD, rows, lane);
            });
            __syncwarp();
        }
        decode_rows<P>(s_warp, lane, d, a.flags, ux, uy, cact);
        }   // float action vectors
        if constexpr (MODE == kSetAction) {
            if (active) {
#pragma unroll
                for (int i = 0; i < A; ++i) a.u[i * n + wi] = make_float2(ux[i], uy[i]);
#pragma unroll
                for (int q = 0; q < NC; ++q) a.c[q * n + wi] = cact[q];
            }
            return;
        }
    }
    if constexpr (MODE == kWorldStep) {
#pragma unroll
        for (int i = 0; i < A; ++i) {
            const float2 v = a.u[i * n + wi];
            ux[i] = v.x; uy[i] = v.y;
        }
#pragma unroll
        for (int q = 0; q < NC; ++q) cact[q] = a.c[q * n + wi];
    }

    if (a.flags & kFlagPdlAfterLoads) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    // ---- World.step (core.py:117-131) --------------------------------------------------------
    if constexpr (MODE == kFusedStep || MODE == kWorldStep) {
        physics<P>(d, w, ux, uy);
#pragma unroll
        for (int q = 0; q < NC; ++q) w.c[q] = cact[q];  // update_agent_state (core.py:171-177)
        if (active) {
#pragma unroll
            for (int i = 0; i < A; ++i)
                if (P::movable(i)) a.pv[i * n + wi] = make_float4(w.px[i], w.py[i], w.vx[i], w.vy[i]);
#pragma unroll
            for (int q = 0; q < NC; ++q) a.comm[q * n + wi] = w.c[q];
        }
        if constexpr (MODE == kWorldStep) return;
    }

    // ---- observation / reward / done / info (environment.py:92-102) -------------------------
    float rew[A];
    float info[(P::INFO > 0 ? P::INFO : 1) * A];
    P::prepare(d, w);   // per-world predicates shared by all agents' observations (world_comm: forest membership)
    P::reward(d, w, rew, (P::INFO > 0 && a.info != nullptr) ? info : nullptr);
    if (a.flags & MPE_FLAG_SHARED_REWARD) {                                      // :100-102 np.sum(reward_n)
        float s = 0.0f;
#pragma unroll
        for (int i = 0; i < A; ++i) s += rew[i];
#pragma unroll
        for (int i = 0; i < A; ++i) rew[i] = s;
    }
    if (!(a.flags & (kFlagPdlEarly | kFlagPdlAfterLoads | kFlagPdlAtExit | kFlagPdlAfterIssue))) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    write_observations<P>(a, d, w, s_warp + Shape<P>::obs_base(), lane, rows, active, w0, wi);
    if (active) {
#pragma unroll
        for (int i = 0; i < A; ++i) {
            a.rew[i * n + wi] = rew[i];
            a.done[i * n + wi] = 0;  // done_callback is None (make_env.py:41-43, environment.py:132-135)
        }
        if (P::INFO > 0 && a.info != nullptr) {
#pragma unroll
            for (int q = 0; q < P::INFO * A; ++q) a.info[q * n + wi] = info[q];
        }
    }
}



// ---- K-step open-loop rollout (SURVEY.md 8(f) rank 3: the persistent multi-step form) --------------------------
// T consecutive MultiAgentEnv.step calls on pre-generated actions act[i] : [T][n_env][act_dim_i] in ONE launch: a
// world's state is loaded once, lives in registers for all T steps and is written once; per step only the actions are
// read (the next step's tiles are prefetched with cp.async while this step computes) and, optionally, the per-step
// rewards written.  Observations are produced for the final state only.  This is what sampling-based planners (CEM /
// MPPI: score many candidate action sequences by their return) and policy evaluation on recorded actions need; HBM
// traffic per env-step drops from 411 B to 60 (+12) B for simple_spread N=3.  Bit-identical to T launches of the
// fused step with rewards summed in step order (tests/test_gpu_api.py).
struct RolloutArgs {
    StepArgs s;
    int32_t T;
    float *rew_steps;   // [T][A][n] per-step rewards (after the shared-reward sum), or null
};

template <class P>
__global__ void __launch_bounds__(kMaxThreads, 1) mpe_rollout_kernel(const __grid_constant__ RolloutArgs ra) {
    constexpr int A = P::A, NC = Shape<P>::kNC;
    const StepArgs &a = ra.s;
    extern __shared__ __align__(16) float smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t n = a.n;
    const int64_t end = a.begin + a.count;
    const int64_t w0 = a.begin + (static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + warp) * 32;
    if (w0 >= end) return;
    const WarpTile wt = warp_tile(lane, n, w0, end);
    const int rows = wt.rows;
    float *s_warp = smem + warp * Shape<P>::kRolloutWarpFloats;
    const DevDesc &d = a.d;
    uintptr_t bits = 0;
#pragma unroll
    for (int i = 0; i < A; ++i) bits |= reinterpret_cast<uintptr_t>(a.act[i]) | static_cast<uintptr_t>((n * P::act_dim(i) * 4) & 15);
    const bool fast = Shape<P>::all_act_dense() && rows == 32 && (bits & 15u) == 0;   // warp-uniform

    auto stage = [&](int t, float *base) {   // action tiles of step t -> base (asynchronously on the fast path)
        static_for<A>([&](auto ic) {
            constexpr int i = decltype(ic)::value;
            constexpr int AD = P::act_dim(i), kVec = 32 * AD / 4;
            const float *g = a.act[i] + (static_cast<int64_t>(t) * n + w0) * AD;
            float *sdst = base + Shape<P>::act_off(i);
            if (fast) {
#pragma unroll
                for (int q0 = 0; q0 < kVec; q0 += 32)
                    if (q0 + 32 <= kVec || q0 + lane < kVec) cp_async16(sdst + 4 * (q0 + lane), g + 4 * (q0 + lane));
            } else {
                tile_load<AD>(sdst, g, rows, lane);
            }
        });
    };
    stage(0, s_warp);
    cp_async_commit();

    typename P::W w;
    load_world<P>(a, wt, w);   // the utterances only matter for T == 0: every step overwrites them

    float rsum[A];
#pragma unroll
    for (int i = 0; i < A; ++i) rsum[i] = 0.0f;
#pragma unroll 1
    for (int t = 0; t < ra.T; ++t) {
        float *cur = s_warp + (t & 1) * Shape<P>::kWarpFloats;           // tiles of step t; step t+1 goes to the other half
        if (t + 1 < ra.T) stage(t + 1, s_warp + ((t + 1) & 1) * Shape<P>::kWarpFloats);
        cp_async_commit();                 // possibly empty: keeps "all but the newest group" == "step t has landed"
        cp_async_wait_group<1>();
        __syncwarp();
        float ux[A], uy[A];
        float cact[NC > 0 ? NC : 1];
        decode_rows<P>(cur, lane, d, a.flags, ux, uy, cact);
        __syncwarp();                      // every lane has read `cur` before step t+2 is staged into it
        physics<P>(d, w, ux, uy);
#pragma unroll
        for (int q = 0; q < NC; ++q) w.c[q] = cact[q];
        rollout_rewards<P>(ra, w, rsum, t, wt);
    }
    cp_async_wait_all();
    if (wt.active) store_world<P>(a, w, wt);
    finish_rollout<P>(a, w, s_warp + Shape<P>::obs_base(), wt, rsum);
}


// ---- K-step CLOSED-LOOP rollout with an in-kernel policy (SURVEY.md 8(f) rank 3, the persistent form with a device-
// resident policy; VERDICT r1 item 9) -------------------------------------------------------------------------------
// T consecutive MultiAgentEnv.step calls in ONE launch where every agent's action is produced inside the kernel by its
// own two-layer perceptron  a_i = softmax(W2_i . relu(W1_i^T . obs_i + b1_i) + b2_i)  (obs_dim_i -> H -> 5 movement
// probabilities, the MADDPG actor shape).  A world's state lives in registers for all T steps; an agent's observation
// is produced straight into registers (never written), pushed through the perceptron (weights of all agents sit in
// shared memory once per block, read as broadcast LDS.128), decoded and integrated.  Per step NOTHING is read from HBM
// and only the optional records (rewards, actions) are written; observations are written for the final state.
// Scenarios whose agents all move and are silent (simple_spread, simple_tag, ...).  The physics / reward / observation
// arithmetic is the fused step's: feeding the recorded actions to T fused steps reproduces the final state, the
// observations and the reward sums bit for bit; the perceptron matches a float64 evaluation to ~1e-6 (tests).
struct PolicyArgs {
    StepArgs s;
    int32_t T;
    float *rew_steps;               // [T][A][n] or null
    float *act_rec[kMaxA];          // [T][n][5] per agent, or null
    const float *w1[kMaxA];         // [obs_dim_i][H]  (input-major: W1^T of a torch Linear(obs_dim_i, H))
    const float *b1[kMaxA];         // [H]
    const float *w2[kMaxA];         // [5][H]          (the layout of a torch Linear(H, 5).weight)
    const float *b2[kMaxA];         // [5]
};

template <class P, int H>
struct PolicyShape {
    __host__ __device__ static constexpr int agent_floats(int i) { return P::obs_dim(i) * H + H + 5 * H + 8; }
    __host__ __device__ static constexpr int agent_off(int i) { int s = 0; for (int j = 0; j < i; ++j) s += agent_floats(j); return s; }
    static constexpr int kWeightFloats = (agent_off(P::A) + 3) & ~3;
};

// observation writer into registers (every index is a compile-time constant after unrolling)
template <int DIM>
struct RegWriter {
    float v[DIM];
    int k = 0;
    __device__ __forceinline__ void put(float x) { v[k++] = x; }
    __device__ __forceinline__ void put2(float a, float b) { v[k] = a; v[k + 1] = b; k += 2; }
    __device__ __forceinline__ void put2(float2 a) { put2(a.x, a.y); }
};


// one agent of the in-kernel policy: observation -> registers -> two-layer perceptron -> softmax -> decoded (u.x, u.y).
// A plain force-inlined function with unrolled loops (not a lambda: arrays captured by reference by a lambda that the
// compiler declines to inline end up in local memory).  W = [W1: OD x H][b1: H][W2: 5 x H][b2: 5] in shared memory.
template <class P, int H, int I>
__device__ __forceinline__ float2 policy_agent(const DevDesc &d, const typename P::W &w, const float *__restrict__ W,
                                               float *__restrict__ record) {
    constexpr int OD = P::obs_dim(I);
    const float *W1 = W, *B1 = W1 + OD * H, *W2 = B1 + H, *B2 = W2 + 5 * H;
    RegWriter<OD> o;
    P::template observe<I>(d, w, o);                       // scenario.observation(agent I) -> registers
    float h[H];
#pragma unroll
    for (int q = 0; q < H; q += 4) {
        const float4 b = *reinterpret_cast<const float4 *>(B1 + q);
        h[q] = b.x; h[q + 1] = b.y; h[q + 2] = b.z; h[q + 3] = b.w;
    }
#pragma unroll
    for (int j = 0; j < OD; ++j) {                         // h += obs[j] * W1[j][:]   (ascending j, FMA)
        const float oj = o.v[j];
#pragma unroll
        for (int q = 0; q < H; q += 4) {
            const float4 wv = *reinterpret_cast<const float4 *>(W1 + j * H + q);
            h[q] = __fmaf_rn(oj, wv.x, h[q]);
            h[q + 1] = __fmaf_rn(oj, wv.y, h[q + 1]);
            h[q + 2] = __fmaf_rn(oj, wv.z, h[q + 2]);
            h[q + 3] = __fmaf_rn(oj, wv.w, h[q + 3]);
        }
    }
#pragma unroll
    for (int q = 0; q < H; ++q) h[q] = fmaxf(h[q], 0.0f);  // ReLU
    float lg[5];
#pragma unroll
    for (int c = 0; c < 5; ++c) {                          // logits[c] = b2[c] + sum_q h[q] * W2[c][q]  (ascending q)
        float acc = B2[c];
#pragma unroll
        for (int q = 0; q < H; q += 4) {
            const float4 wv = *reinterpret_cast<const float4 *>(W2 + c * H + q);
            acc = __fmaf_rn(h[q], wv.x, acc);
            acc = __fmaf_rn(h[q + 1], wv.y, acc);
            acc = __fmaf_rn(h[q + 2], wv.z, acc);
            acc = __fmaf_rn(h[q + 3], wv.w, acc);
        }
        lg[c] = acc;
    }
    const float m = fmaxf(fmaxf(fmaxf(lg[0], lg[1]), fmaxf(lg[2], lg[3])), lg[4]);
    float e[5], sum = 0.0f;
#pragma unroll
    for (int c = 0; c < 5; ++c) { e[c] = expf(__fsub_rn(lg[c], m)); sum = __fadd_rn(sum, e[c]); }
    float pr[5];
#pragma unroll
    for (int c = 0; c < 5; ++c) pr[c] = __fdiv_rn(e[c], sum);                // softmax: the action vector
    if (record != nullptr) {
#pragma unroll
        for (int c = 0; c < 5; ++c) record[c] = pr[c];
    }
    return movement_force(pr[1], pr[2], pr[3], pr[4], d.a_sens[I]);   // _set_action, as decode_rows
}

template <class P, int H>
__global__ void __launch_bounds__(128) mpe_policy_rollout_kernel(const __grid_constant__ PolicyArgs pa) {
    static_assert(P::NS == 0 && H % 4 == 0, "policy rollout: silent agents, hidden width a multiple of 4");
    constexpr int A = P::A;
    using PS = PolicyShape<P, H>;
    const StepArgs &a = pa.s;
    extern __shared__ __align__(16) float smem[];
    float *s_w = smem;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // ---- all agents' weights -> shared memory, once per block ------------------------------------------------
    static_for<A>([&](auto ic) {
        constexpr int i = decltype(ic)::value;
        constexpr int OD = P::obs_dim(i);
        float *base = s_w + PS::agent_off(i);
        for (int q = threadIdx.x; q < OD * H; q += blockDim.x) base[q] = pa.w1[i][q];
        for (int q = threadIdx.x; q < H; q += blockDim.x) base[OD * H + q] = pa.b1[i][q];
        for (int q = threadIdx.x; q < 5 * H; q += blockDim.x) base[OD * H + H + q] = pa.w2[i][q];
        for (int q = threadIdx.x; q < 5; q += blockDim.x) base[OD * H + H + 5 * H + q] = pa.b2[i][q];
    });
    __syncthreads();

    const int64_t n = a.n;
    const int64_t end = a.begin + a.count;
    const int64_t w0 = a.begin + (static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + warp) * 32;
    if (w0 >= end) return;
    const WarpTile wt = warp_tile(lane, n, w0, end);
    float *s_warp = smem + PS::kWeightFloats + warp * Shape<P>::kWarpFloats;
    const DevDesc &d = a.d;

    typename P::W w;
    load_world<P>(a, wt, w);

    float rsum[A];
#pragma unroll
    for (int i = 0; i < A; ++i) rsum[i] = 0.0f;
#pragma unroll 1
    for (int t = 0; t < pa.T; ++t) {
        float ux[A], uy[A];
        P::prepare(d, w);
        static_for<A>([&](auto ic) {
            constexpr int i = decltype(ic)::value;
            const float2 u = policy_agent<P, H, i>(d, w, s_w + PolicyShape<P, H>::agent_off(i),
                                                   (pa.act_rec[i] != nullptr && wt.active)
                                                       ? pa.act_rec[i] + (static_cast<int64_t>(t) * n + wt.wi) * 5 : nullptr);
            ux[i] = u.x;
            uy[i] = u.y;
        });
        physics<P>(d, w, ux, uy);
        rollout_rewards<P>(pa, w, rsum, t, wt);
    }
    if (wt.active) store_world<P>(a, w, wt);
    finish_rollout<P>(a, w, s_warp + Shape<P>::obs_base(), wt, rsum);
}

template <class P>
constexpr bool policy_rollout_ok() {     // every agent moves, nobody speaks: the action is the 5-vector of probabilities
    bool ok = P::NS == 0;
    for (int i = 0; i < P::A; ++i) ok = ok && P::movable(i) && P::act_dim(i) == 5;
    return ok;
}
// built for the BASELINE.json worlds (each instantiation unrolls obs_dim x H FMAs per agent: compile time)
template <class P> struct PolicyBuilt { static constexpr bool value = false; };
template <> struct PolicyBuilt<Simple<1, 1>> { static constexpr bool value = true; };
template <> struct PolicyBuilt<Spread<3>> { static constexpr bool value = true; };
template <> struct PolicyBuilt<Tag<3, 1, 2>> { static constexpr bool value = true; };
// the two-hidden-layer actor (mpe_policy_mlp_rollout_kernel) is built for those and for the reference's default
// configurations of the scenarios with speaking or immovable agents
template <class P> struct MlpBuilt : PolicyBuilt<P> {};
template <> struct MlpBuilt<SpeakerListener> { static constexpr bool value = true; };
template <> struct MlpBuilt<Reference> { static constexpr bool value = true; };
template <> struct MlpBuilt<Crypto> { static constexpr bool value = true; };
template <> struct MlpBuilt<Adversary<1, 2, 2>> { static constexpr bool value = true; };
template <> struct MlpBuilt<Push<1, 1, 2>> { static constexpr bool value = true; };
// ... and for the entity-count variants the scenario kwargs reach (movable, silent agents with 5-entry actions)
template <> struct MlpBuilt<Spread<2>> { static constexpr bool value = true; };
template <> struct MlpBuilt<Spread<4>> { static constexpr bool value = true; };
template <> struct MlpBuilt<Spread<5>> { static constexpr bool value = true; };
template <> struct MlpBuilt<Spread<6>> { static constexpr bool value = true; };
template <> struct MlpBuilt<Tag<1, 1, 2>> { static constexpr bool value = true; };
template <> struct MlpBuilt<Tag<2, 1, 2>> { static constexpr bool value = true; };
template <> struct MlpBuilt<Tag<4, 2, 2>> { static constexpr bool value = true; };
template <> struct MlpBuilt<Tag<6, 2, 3>> { static constexpr bool value = true; };
template <> struct MlpBuilt<Adversary<1, 3, 3>> { static constexpr bool value = true; };

// ---- initial conditions of one world (e.g. simple_spread.py:31-45, simple_tag.py:45-53) -----------------------------
// Agents ~ U(-1, 1)^2 at rest (immovable ones too), landmarks ~ U(-landmark_range, landmark_range)^2, comm 0, goal g =
// word g of Philox block 0x80000000 mod goal_mod.  One Philox4x32-10 block = 4 x 32 bits = two entities' (x, y), entities
// in the order agents then landmarks; key = seed, counter = (global world index lo, hi, low 32 bits of epoch, block).
// The one definition of a reset: reset_kernel writes the draw to the state arrays, the episode form of the MLP rollout
// to the world's registers, through `out` (agent(i, x, y), landmark(l, x, y), comm(q), goal(g, v)).
__host__ __device__ constexpr float reset_landmark_range(int scenario) {   // simple_tag.py:53, simple_world_comm.py:105-113
    return (scenario == MPE_SCN_TAG || scenario == MPE_SCN_WORLD_COMM) ? 0.9f : 1.0f;
}
template <class Out>
__device__ __forceinline__ void draw_initial_state(int A, int L, int NC, int G, uint64_t seed, uint64_t gw, uint64_t epoch,
                                                   float landmark_range, uint32_t goal_mod, Out &out) {
    const uint2 key = make_uint2(static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
    const int E = A + L;
#pragma unroll
    for (int e = 0; e < E; e += 2) {
        const uint4 r = philox4x32_10(make_uint4(static_cast<uint32_t>(gw), static_cast<uint32_t>(gw >> 32),
                                                 static_cast<uint32_t>(epoch), static_cast<uint32_t>(e >> 1)), key);
        const uint32_t bits[4] = {r.x, r.y, r.z, r.w};
        for (int k = 0; k < 2 && e + k < E; ++k) {
            const int ent = e + k;
            if (ent < A) {
                out.agent(ent, uniform_from_bits(bits[2 * k], -1.0f, 1.0f), uniform_from_bits(bits[2 * k + 1], -1.0f, 1.0f));
            } else {
                out.landmark(ent - A, uniform_from_bits(bits[2 * k], -landmark_range, landmark_range),
                             uniform_from_bits(bits[2 * k + 1], -landmark_range, landmark_range));
            }
        }
    }
#pragma unroll
    for (int q = 0; q < NC; ++q) out.comm(q);
    if (G > 0) {
        const uint4 r = philox4x32_10(make_uint4(static_cast<uint32_t>(gw), static_cast<uint32_t>(gw >> 32),
                                                 static_cast<uint32_t>(epoch), 0x80000000u), key);
        const uint32_t bits[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
        for (int g = 0; g < G && g < 4; ++g) out.goal(g, static_cast<int32_t>(bits[g] % goal_mod));
    }
}


// ---- K-step closed-loop rollout with MADDPG's two-hidden-layer actor on the tensor cores ---------------------------
// The persistent structure of mpe_policy_rollout_kernel (state in registers for all T steps, nothing read from HBM per
// step, the same physics<P> / P::reward / P::observe<I>) with the MADDPG actor (mlp_model)
//     logits_i = W3_i relu(W2_i relu(W1_i obs_i + b1_i) + b2_i) + b3_i       obs_dim_i -> H -> H -> act_dim_i,  H = 32 or 64
// evaluated by the warp as three TF32 GEMMs with mma.sync.m16n8k8 (fp32 accumulation):
//     [32 x K1] . [K1 x H] -> ReLU -> [32 x H] . [H x H] -> ReLU -> [32 x H] . [H x NOUT_i],  NOUT_i = act_dim_i rounded up to 8
// One warp = 32 worlds = two m16 tiles.  Each lane writes its observation row into the warp's observation tile (the
// layout of the fused step's coalesced tile store, ObsTile<obs_dim>); the A fragments are read from it with the columns
// at and beyond obs_dim read as zero, so K1 = obs_dim rounded up to 8.  The accumulators of one layer are the A fragments
// of the next without any data movement: within a k-tile a lane holds hidden units 2q and 2q+1 of rows g and g+8 and
// the next layer's B fragments are staged with the same permutation of k.  Layers 2 and 3 are interleaved per 8-unit
// tile of h2, so h2 never exists as a whole.  The act_dim_i logits (padded to NOUT_i) go back to their lane through a
// small shared-memory tile; that lane does the softmax (or the Gumbel-softmax sample), the _set_action decode and the
// step.
// Action sub-spaces (environment.py:40-66, MADDPG's SoftMultiCategoricalPd): the logits split, in action-vector order,
// into 5 movement logits if the agent is movable, then dim_c utterance logits if it speaks; the action is the
// concatenation of one softmax per sub-space.  Movement is decoded as _set_action does; an utterance becomes the
// world's comm state after the physics (update_agent_state), as in the fused step, so the other agents observe it from
// step t + 1 on.  Immovable agents keep their position and velocity.
// Rounding: every tensor-core operand -- observations, h1, h2 and all weights -- is converted with cvt.rna.tf32.f32
// (round to nearest, ties away from zero, to 10 mantissa bits); the weights once, while they are staged.  Biases are
// the accumulators' fp32 initial values.
// Exploration (explore != 0): agent i at step t acts with one softmax(z - log(-log u)) per sub-space
// (SoftCategoricalPd.sample), in fp32 with logf.  Logit k of the action vector uses u_k = word k mod 4 of Philox4x32-10
// block b = k div 4, with key = explore_seed and counter = (global world index lo, hi, low 32 bits of explore_epoch,
// kExploreTag | ((t * A + i) * S + b)), S = mlp_explore_stride<P>() blocks per agent and step; u = ((bits >> 8) + 0.5)
// * 2^-24 with the sum rounded toward zero in fp32 (exact below 2^23, the half is dropped above), so u lies in
// [2^-25, 1 - 2^-24].  The tag bit keeps this stream apart from reset_kernel's counters, so an exploration seed equal
// to the env seed does not correlate the noise with initial positions; the global world index (world_offset + w) makes
// the noise independent of sharding.
constexpr uint32_t kExploreTag = 0x40000000u;
// S: 2 blocks (8 uniforms) per agent and step when every action vector has at most 8 entries, else 4 (simple_reference:
// 15).  S = 2 for the 5-logit programs keeps their stream what it has always been.
template <class P>
__host__ __device__ constexpr int mlp_max_act_dim() { int m = 0; for (int i = 0; i < P::A; ++i) m = P::act_dim(i) > m ? P::act_dim(i) : m; return m; }
template <class P>
__host__ __device__ constexpr int mlp_explore_stride() { return mlp_max_act_dim<P>() <= 8 ? 2 : 4; }

struct MlpPolicyArgs {
    StepArgs s;
    int32_t T;
    int32_t explore;
    uint64_t seed, epoch, world_offset;
    float *rew_steps;               // [T][A][n] or null
    float *act_rec[kMaxA];          // [T][n][act_dim_i] per agent, or null: the action applied (sampled when exploring)
    float *obs_rec[kMaxA];          // [T][n][obs_dim_i] per agent, or null: the observation the actor saw at step t
    const float *w1[kMaxA], *b1[kMaxA];   // torch nn.Linear layout: [H][obs_dim_i], [H]
    const float *w2[kMaxA], *b2[kMaxA];   // [H][H], [H]
    const float *w3[kMaxA], *b3[kMaxA];   // [act_dim_i][H], [act_dim_i]
};
static_assert(sizeof(MlpPolicyArgs) <= 4096, "kernel parameter space");

// Episode form (mpe_policy_mlp_episode_kernel): `episodes` episodes of p.T steps in one launch.  After the last step of
// episode e the world is redrawn as reset_kernel draws it with (reset_seed, global world index, reset_epoch + e); the
// exploration of episode e uses epoch p.epoch + e and restarts its step counter at 0.  Records are indexed by the
// global step e * p.T + t, and p.s.rew receives the per-episode returns [episodes][A][n].
struct MlpEpisodeArgs {
    MlpPolicyArgs p;
    float2 *lm;                     // p.s.lm and p.s.goal, writable: every episode end redraws them
    int32_t *goal;
    int32_t episodes;
    uint64_t reset_seed, reset_epoch;
    float *final_obs[kMaxA];        // [episodes][n][obs_dim_i] per agent, or null: the observation after the last step
};
static_assert(sizeof(MlpEpisodeArgs) <= 4096, "kernel parameter space");

// Categorical form (CATEGORICAL): the policy-gradient action.  Per sub-space the agent applies the one-hot vector of
// k = argmax_c (z_c - log(-log u_c)) when exploring (the same u as the Gumbel-softmax sample), k = argmax_c z_c when not,
// the lowest index winning ties; k is the position in the logit segment (the one-hot convention, environment.py:173-175),
// not the discrete_action_input code.  The log-probability of the agent's action is the sum over its sub-spaces, in
// order, of log_softmax(z)[k] = (z_k - m) - log(sum_c exp(z_c - m)), m the maximum of the unperturbed segment.  The
// records live next to, not inside, MlpPolicyArgs / MlpEpisodeArgs so that the default kernels' parameters keep their
// layout; p.act_rec is null in this form.
struct MlpCategoricalRecords {
    int32_t *index[kMaxA];          // [T][n][n_sub_i] per agent, or null: k of each sub-space, movement first
    float *logp;                    // [T][A][n] or null: the log-probability of the action applied
};
struct MlpCategoricalArgs {
    MlpPolicyArgs p;
    MlpCategoricalRecords c;
};
struct MlpCategoricalEpisodeArgs {
    MlpEpisodeArgs e;
    MlpCategoricalRecords c;
};
static_assert(sizeof(MlpCategoricalEpisodeArgs) <= 4096, "kernel parameter space");

// MAPPO's MLP actor (MAPPO, MLPBase with layer_N = 1 and its categorical ACTLayer head), categorical form only, H = 64:
//     [LN(obs_dim_i)] -> Linear(obs_dim_i, 64) -> act -> LN(64) -> Linear(64, 64) -> act -> LN(64) -> Linear(64, act_dim_i)
// act is ReLU or tanh.  Every LayerNorm's affine (gamma, beta) is folded into the Linear after it on the host
// (W' = W diag(gamma), b' = b + W beta), so w1..b3 are the folded network and the kernel applies parameter-free
// normalisation (x - mu) * rsqrt(var + eps) with two-pass fp32 statistics (mlp_agent).
enum : uint32_t { kMappoFeatureNorm = 1u, kMappoTanh = 2u };
struct MlpMappoArgs {
    MlpCategoricalArgs c;
    float eps;                      // of every LayerNorm
    uint32_t net_flags;             // kMappoFeatureNorm: the input LayerNorm; kMappoTanh: tanh instead of ReLU
};
struct MlpMappoEpisodeArgs {
    MlpCategoricalEpisodeArgs c;
    float eps;
    uint32_t net_flags;
};
static_assert(sizeof(MlpMappoEpisodeArgs) <= 4096, "kernel parameter space");

// MAPPO's recurrent actor (rMAPPO's R_Actor: MLPBase -> RNNLayer -> categorical ACTLayer, recurrent_N = 1), one weight
// set shared by every agent (share_policy), categorical form only, H = 64:
//     [LN(obs_dim)] -> Linear(obs_dim, 64) -> act -> LN(64) -> Linear(64, 64) -> act -> LN(64) = x
//     h' = GRU(x, h) (torch's gate order r, z, n) -> LN(64) -> Linear(64, act_dim)
// The base's LayerNorms fold as MAPPO's do; the base's last LayerNorm folds into W_ih, b_ih and the GRU's LayerNorm into
// the head.  w1..b3 of MlpPolicyArgs hold the base and the head (every agent's pointer the same); the GRU's weights
// (torch layout, W [192][64], b [192]) and the hidden state live here.  h is [A][n][64]: read at every agent's turn,
// written back with h' (the state after the last step when the kernel ends), except that in the episode form every
// episode starts from h = 0 (MAPPO's mask after done).  h_rec ([T][A][n][64] or null) receives the h each step's
// actor consumed.
struct MlpGruState {
    const float *w_ih, *b_ih, *w_hh, *b_hh;
    float *h;
    float *h_rec;
};
struct MlpGruArgs {
    MlpMappoArgs m;
    MlpGruState g;
};
struct MlpGruEpisodeArgs {
    MlpMappoEpisodeArgs m;
    MlpGruState g;
};
static_assert(sizeof(MlpGruEpisodeArgs) <= 4096, "kernel parameter space");
// Per-agent recurrent actors (mpe_policy_gru_separated[_episode]_kernel): g's state as the shared actor's, agent i's
// weights in its fragment image at images + GruSeparatedShape::image_off(i) (written by mpe_gru_image_kernel); the
// weight pointers of g are not read.
struct MlpGruSeparatedArgs {
    MlpGruArgs g;
    const float *images;
};
struct MlpGruSeparatedEpisodeArgs {
    MlpGruEpisodeArgs g;
    const float *images;
};
static_assert(sizeof(MlpGruSeparatedEpisodeArgs) <= 4096, "kernel parameter space");
// The fragment images' sources: w[j][i] is agent i's W1, b1, W2, b2, W_ih, b_ih, W_hh, b_hh, W3, b3 (j = 0 .. 9,
// folded as the shared actor's, torch layouts)
struct GruImageArgs {
    const float *w[10][kMaxA];
    float *images;
};

// MAPPO's centralized critic (R_Critic with use_centralized_V, recurrent off: MLPBase with layer_N = 1, then v_out) next
// to MAPPO's actor:
//     [LN(D)] -> Linear(D, 64) -> act -> LN(64) -> Linear(64, 64) -> act -> LN(64) -> Linear(64, 1)
// Its input is share_obs, every agent's raw observation concatenated in agent order (D = sum of obs_dim_i); act, eps
// and the input LayerNorm are the actor's (MlpMappoArgs), the affines folded as the actor's.  count = 1: one shared
// critic (w*[0]), its value written for every agent; count = A: agent i's critic (w*[i]) evaluates the same input.
// values [T][A][n] receives V of the state each step's actors act on (MAPPO's value_preds), final_values [A][n] (in the
// episode form [episodes][A][n]) V of the state after the last step (of each episode, before its reset).
struct MlpCriticState {
    const float *w1[kMaxA], *b1[kMaxA];   // [64][D], [64]
    const float *w2[kMaxA], *b2[kMaxA];   // [64][64], [64]
    const float *w3[kMaxA], *b3[kMaxA];   // [1][64], [1]
    int32_t count;
    float *values, *final_values;
};
struct MlpCriticArgs {
    MlpMappoArgs m;
    MlpCriticState v;
};
struct MlpCriticEpisodeArgs {
    MlpMappoEpisodeArgs m;
    MlpCriticState v;
};
static_assert(sizeof(MlpCriticEpisodeArgs) <= 4096, "kernel parameter space");

template <class P, int H>
struct MlpShape {
    static constexpr int NT = H / 8;                                   // n-tiles of a hidden layer (= its k-tiles)
    __host__ __device__ static constexpr int kt1(int i) { return (P::obs_dim(i) + 7) / 8; }
    __host__ __device__ static constexpr int nout(int i) { return (P::act_dim(i) + 7) / 8 * 8; }   // layer-3 columns
    // per agent, in floats: B fragments [k-tile][n-tile][lane][2] of W1, W2, W3, then b1 [H], b2 [H], b3 [NOUT]; the
    // rows of W3 and b3 at and beyond act_dim are zero
    __host__ __device__ static constexpr int w2_off(int i) { return 64 * kt1(i) * NT; }
    __host__ __device__ static constexpr int w3_off(int i) { return w2_off(i) + 64 * NT * NT; }
    __host__ __device__ static constexpr int b1_off(int i) { return w3_off(i) + 64 * NT * (nout(i) / 8); }
    __host__ __device__ static constexpr int b2_off(int i) { return b1_off(i) + H; }
    __host__ __device__ static constexpr int b3_off(int i) { return b2_off(i) + H; }
    __host__ __device__ static constexpr int agent_floats(int i) { return b3_off(i) + nout(i); }
    __host__ __device__ static constexpr int agent_off(int i) { int s = 0; for (int j = 0; j < i; ++j) s += agent_floats(j); return s; }
    static constexpr int kWeightFloats = agent_off(P::A);
    // per warp: [observation tile][logit tile 32 x (max NOUT + 1)]; the final observations are written through the
    // same tile.  The odd pitch keeps each lane's row reads conflict-free.
    __host__ __device__ static constexpr int obs_tile_floats() { int m = 0; for (int i = 0; i < P::A; ++i) m = 32 * Shape<P>::obs_pitch(i) > m ? 32 * Shape<P>::obs_pitch(i) : m; return (m + 3) & ~3; }
    __host__ __device__ static constexpr int max_nout() { int m = 0; for (int i = 0; i < P::A; ++i) m = nout(i) > m ? nout(i) : m; return m; }
    static constexpr int kLogitPitch = max_nout() + 1;
    static constexpr int kLogitOff = obs_tile_floats();
    static constexpr int kWarpFloats = (kLogitOff + 32 * kLogitPitch + 3) & ~3;
    static_assert(Shape<P>::kWarpFloats - Shape<P>::obs_base() <= kLogitOff, "final observations fit the tile");
};

// Warps per block at most: one copy of the weights serves all of them, and with 6-212 KB of weights one block is what
// fits an SM, so this is also the residency.  The smaller of two limits:
//  - registers (mlp_register_warps): a block's warps share the four SM sub-partitions' 16 K registers each, so 16 warps
//    leave 128 registers per thread, 9-12 warps 168 and 8 or fewer 255.  Blocks are 16 warps unless that spills
//    (ptxas -v): then 12, or 8 where 168 spills too.  At H = 64 every program with four or more agents (their state
//    next to the 64 registers of h1) and simple_reference (two 8-column logit tiles and 20 comm floats next to h1)
//    take 12; the exceptions below are the rest.  The episode form adds the reset draw and the episode-end stores, the
//    categorical form the arg-max, the log-probability and the index stores, and MAPPO's actor a second 32-register
//    m-tile of h2 next to h1 for its LayerNorms (see mlp_agent), so an exception names the forms it holds for.
//  - shared memory (mlp_smem_warps): the weights plus kWarpFloats per warp within the 227 KB a block may opt in to on
//    H100.  Below the register limit only for tag 6+2 at H = 64 (212 KB of weights, 3 warps).
// The forms, indexed by episodes | kind << 1 with kind 0 for softmax actions, 1 for categorical ones and 2 for MAPPO's
// actor (categorical records, H = 64 only), and the masks an exception lists them by
enum : int { kMlpForms = 6, kFormS = 1, kFormE = 2, kFormC = 4, kFormCE = 8, kFormM = 16, kFormME = 32, kFormAll = 63 };
template <int FORMS, int WARPS>
struct MlpException { static constexpr int forms = FORMS, warps = WARPS; };
// One exception per (program, H), so that no kernel matches two: a second one would redefine the specialisation.  The
// stack ptxas -v showed without it, by form: MADDPG's (S, E, C, CE), then MAPPO's (M, ME)
template <class P, int H> struct MlpRegisterException : MlpException<0, 0> {};
template <> struct MlpRegisterException<Spread<2>, 64> : MlpException<kFormAll, 12> {};      // 8 bytes at 128; M, ME 16, 24 at 128
template <> struct MlpRegisterException<Tag<1, 1, 2>, 64> : MlpException<kFormAll, 12> {};   // 8 at 128; M, ME 16, 24 at 128
template <> struct MlpRegisterException<Tag<2, 1, 2>, 64> : MlpException<kFormAll, 12> {};   // 8 at 128; M, ME 56, 56 at 128
template <> struct MlpRegisterException<Spread<6>, 64> : MlpException<kFormAll, 8> {};       // 16 at 168; M, ME 64, 56 at 168
template <> struct MlpRegisterException<Spread<6>, 32> : MlpException<kFormAll, 12> {};      // 48 at 128
template <> struct MlpRegisterException<Tag<4, 2, 2>, 32> : MlpException<kFormAll, 12> {};   // 16 at 128
template <> struct MlpRegisterException<Tag<6, 2, 3>, 32> : MlpException<kFormAll, 8> {};    // 64 at 128, 8 at 168
template <> struct MlpRegisterException<SpeakerListener, 64>
    : MlpException<kFormE | kFormCE | kFormM | kFormME, 12> {};                                 // 8 at 128; M, ME 16, 16 at 128
template <> struct MlpRegisterException<Adversary<1, 2, 2>, 64>
    : MlpException<kFormE | kFormCE | kFormM | kFormME, 12> {};                                 // 16 at 128; M, ME 32, 40 at 128
template <> struct MlpRegisterException<Reference, 64> : MlpException<kFormE | kFormCE, 8> {};             // 8 at 168
template <> struct MlpRegisterException<Tag<4, 2, 2>, 64> : MlpException<kFormE | kFormCE, 8> {};          // 8 at 168
template <> struct MlpRegisterException<Spread<3>, 64>
    : MlpException<kFormE | kFormC | kFormCE | kFormM | kFormME, 12> {};                        // 8 at 128; M, ME 32, 32 at 128
template <> struct MlpRegisterException<Push<1, 1, 2>, 64> : MlpException<kFormC | kFormCE, 12> {};        // 8 at 128
template <> struct MlpRegisterException<Crypto, 64> : MlpException<kFormCE | kFormM, 12> {};               // 16 at 128; M 8 at 128
template <> struct MlpRegisterException<Spread<4>, 64> : MlpException<kFormCE, 8> {};                      // 8 at 168
template <class P, int H>
__host__ __device__ constexpr int mlp_register_rule() { return (H == 64 && (P::A >= 4 || mlp_max_act_dim<P>() > 8)) ? 12 : 16; }
template <class P, int H, int FORM>
__host__ __device__ constexpr int mlp_register_warps() {
    using X = MlpRegisterException<P, H>;
    return (X::forms >> FORM & 1) ? X::warps : mlp_register_rule<P, H>();
}
constexpr int kMlpSmemBytes = 232448;
template <class P, int H>
__host__ __device__ constexpr int mlp_smem_warps() {
    return (kMlpSmemBytes / 4 - MlpShape<P, H>::kWeightFloats) / MlpShape<P, H>::kWarpFloats;
}
template <class P, int H, int FORM>
__host__ __device__ constexpr int mlp_block_warps() {
    constexpr int r = mlp_register_warps<P, H, FORM>(), s = mlp_smem_warps<P, H>();
    return r < s ? r : s;
}
// the two programs whose weights fill most of the 227 KB
static_assert(MlpShape<Spread<6>, 64>::kWeightFloats * 4 == 175296 && MlpShape<Spread<6>, 64>::kWarpFloats * 4 == 6016 &&
              mlp_smem_warps<Spread<6>, 64>() == 9, "spread N=6, H = 64: 175 296 + 9 x 6016 = 229 440 B");
static_assert(MlpShape<Tag<6, 2, 3>, 64>::kWeightFloats * 4 == 217344 && MlpShape<Tag<6, 2, 3>, 64>::kWarpFloats * 4 == 4992 &&
              mlp_smem_warps<Tag<6, 2, 3>, 64>() == 3, "tag 6+2, H = 64: 217 344 + 3 x 4992 = 232 320 B");

// The recurrent actor (MlpGruArgs) is built for the programs whose agents all observe and act alike, which one shared
// policy needs: simple, simple_spread N = 2..6 and simple_reference.
template <class P> struct GruBuilt { static constexpr bool value = false; };
template <> struct GruBuilt<Simple<1, 1>> { static constexpr bool value = true; };
template <> struct GruBuilt<Spread<2>> { static constexpr bool value = true; };
template <> struct GruBuilt<Spread<3>> { static constexpr bool value = true; };
template <> struct GruBuilt<Spread<4>> { static constexpr bool value = true; };
template <> struct GruBuilt<Spread<5>> { static constexpr bool value = true; };
template <> struct GruBuilt<Spread<6>> { static constexpr bool value = true; };
template <> struct GruBuilt<Reference> { static constexpr bool value = true; };

// One weight set in shared memory, in floats: B fragments [k-tile][n-tile][lane][2] of W1, W2, W_ih (24 n-tiles: r, z,
// n), W_hh, the head W3, then b1 [64], b2 [64], b_ih [192], b_hh [192], b3 [NOUT].  Per warp the MLP actor's
// observation and logit tiles: h and h' stay in registers (one m-tile at a time, see mlp_agent).  GruAgentShape is the
// layout for agent I's obs_dim and act_dim; GruShape, the one shared set, is agent 0's.
template <class P, int I>
struct GruAgentShape {
    using M = MlpShape<P, 64>;
    static constexpr int NT = 8, NG = 24;
    static constexpr int w2_off = 64 * M::kt1(I) * NT;
    static constexpr int wih_off = w2_off + 64 * NT * NT;
    static constexpr int whh_off = wih_off + 64 * NT * NG;
    static constexpr int w3_off = whh_off + 64 * NT * NG;
    static constexpr int b1_off = w3_off + 64 * NT * (M::nout(I) / 8);
    static constexpr int b2_off = b1_off + 64;
    static constexpr int bih_off = b2_off + 64;
    static constexpr int bhh_off = bih_off + 192;
    static constexpr int b3_off = bhh_off + 192;
    static constexpr int kWeightFloats = b3_off + M::nout(I);
    static constexpr int kImageFloats = (kWeightFloats + 3) & ~3;   // a fragment image: padded to 16 bytes
};
template <class P>
struct GruShape : GruAgentShape<P, 0> {
    static constexpr bool shared_ok() {
        for (int i = 1; i < P::A; ++i)
            if (P::obs_dim(i) != P::obs_dim(0) || P::act_dim(i) != P::act_dim(0)) return false;
        return true;
    }
    static_assert(shared_ok(), "one shared policy: every agent observes and acts alike");
    static constexpr int kWarpFloats = MlpShape<P, 64>::kWarpFloats;
};
static_assert(GruShape<Simple<1, 1>>::kWeightFloats * 4 == 120864, "simple: 120 864 B of weights");
static_assert(GruShape<Spread<3>>::kWeightFloats * 4 == 124960, "spread N=3: 124 960 B");
static_assert(GruShape<Reference>::kWeightFloats * 4 == 127040, "simple_reference: 127 040 B");
static_assert(GruShape<Spread<6>>::kWeightFloats * 4 == 129056, "spread N=6: 129 056 B");
// Warps per block, both forms and every program: 8, which leaves 255 registers per thread -- x, h (TF32) and h' of one
// m-tile are 96 of them next to 16 gate accumulators, the world state and the logits (ptxas -v: no stack, 164-252
// registers).  One block per SM: the weights take more than half of its shared memory.
constexpr int kGruWarps = 8;
template <class P>
__host__ __device__ constexpr int gru_block_warps() {
    static_assert((GruShape<P>::kWeightFloats + kGruWarps * GruShape<P>::kWarpFloats) * 4 <= kMlpSmemBytes,
                  "8 warps' tiles fit next to the weights");
    return kGruWarps;
}

// Per-agent recurrent actors (rMAPPO's separated runner: agent i's own R_Actor, MlpGruSeparatedArgs) are built for the
// programs whose agents observe or act differently, where one shared policy cannot serve: simple_speaker_listener.
template <class P> struct GruSeparatedBuilt { static constexpr bool value = false; };
template <> struct GruSeparatedBuilt<SpeakerListener> { static constexpr bool value = true; };
// Every agent's weight set does not fit in shared memory at once (speaker_listener: 120 864 + 122 912 B against 232 448
// B), so the block keeps one slot, sized for the largest agent, and restages it at every agent's turn from agent i's
// fragment image: GruAgentShape<P, i>'s layout, prepared once per call in a global workspace, images back to back.
template <class P>
struct GruSeparatedShape {
    using M = MlpShape<P, 64>;
    // GruAgentShape<P, i>::kImageFloats for a run-time i (gru_image checks the two agree)
    __host__ __device__ static constexpr int image_floats(int i) {
        return (64 * 8 * (M::kt1(i) + 8 + 2 * 24 + M::nout(i) / 8) + 64 + 64 + 192 + 192 + M::nout(i) + 3) & ~3;
    }
    __host__ __device__ static constexpr int image_off(int i) { int s = 0; for (int j = 0; j < i; ++j) s += image_floats(j); return s; }
    static constexpr int kImagesFloats = image_off(P::A);
    __host__ __device__ static constexpr int slot_floats() { int m = 0; for (int i = 0; i < P::A; ++i) m = image_floats(i) > m ? image_floats(i) : m; return m; }
    static constexpr int kSlotFloats = slot_floats();
};
template <class P>
__host__ __device__ constexpr int gru_separated_block_warps() {
    static_assert((GruSeparatedShape<P>::kSlotFloats + kGruWarps * MlpShape<P, 64>::kWarpFloats) * 4 <= kMlpSmemBytes,
                  "8 warps' tiles fit next to the slot");
    return kGruWarps;
}
static_assert(GruSeparatedShape<SpeakerListener>::image_floats(0) * 4 == 120864 &&
              GruSeparatedShape<SpeakerListener>::image_floats(1) * 4 == 122912 &&
              GruSeparatedShape<SpeakerListener>::kImagesFloats * 4 == 243776,
              "speaker_listener: a 120 864 B speaker and a 122 912 B listener, 243 776 B together");
static_assert((GruSeparatedShape<SpeakerListener>::kSlotFloats + kGruWarps * MlpShape<SpeakerListener, 64>::kWarpFloats) * 4 ==
              143392, "speaker_listener: a 122 912 B slot and 8 warps' 2 560 B tiles");

// One critic's weights in shared memory, in floats: B fragments [k-tile][n-tile][lane][2] of W1, agent by agent (agent
// i's obs_dim_i columns zero-padded to whole k-tiles, so that layer 1 is a sum of k-slices over the agents'
// observation tiles), then of W2 and W3 (one n-tile, its one real column first), then b1 [64], b2 [64], b3 [8].  They
// follow the actor's weights (MlpShape), count sets in a row; the warps' tiles are the actor's.  K >= 0 is IPPO's local
// critic of agent K, whose input is obs_K alone: W1 has agent K's k-tiles only, at offset 0.
template <class P, int K = -1>
struct CriticShape {
    using M = MlpShape<P, 64>;
    static constexpr int NT = 8;
    __host__ __device__ static constexpr int in_dim() {
        if (K >= 0) return P::obs_dim(K);
        int s = 0; for (int i = 0; i < P::A; ++i) s += P::obs_dim(i); return s;
    }
    __host__ __device__ static constexpr int col_off(int i) {
        if (K >= 0) return 0;
        int s = 0; for (int j = 0; j < i; ++j) s += P::obs_dim(j); return s;
    }
    __host__ __device__ static constexpr int w1_off(int i) {
        if (K >= 0) return 0;
        int s = 0; for (int j = 0; j < i; ++j) s += 64 * M::kt1(j) * NT; return s;
    }
    static constexpr int w2_off = K >= 0 ? 64 * M::kt1(K) * NT : w1_off(P::A);
    static constexpr int w3_off = w2_off + 64 * NT * NT;
    static constexpr int b1_off = w3_off + 64 * NT;
    static constexpr int b2_off = b1_off + 64;
    static constexpr int b3_off = b2_off + 64;
    static constexpr int kFloats = b3_off + 8;
};
// Warps per block at most, for the critics' count: the weights of the actor and of `count` critics plus kWarpFloats per
// warp within the 227 KB
template <class P>
__host__ __device__ constexpr int critic_smem_warps(int count) {
    return (kMlpSmemBytes / 4 - MlpShape<P, 64>::kWeightFloats - count * CriticShape<P>::kFloats) / MlpShape<P, 64>::kWarpFloats;
}
// The critic is built where one shared critic leaves room for a warp: every MAPPO program but spread N=6 (175 KB of
// actor weights and an 80 KB critic) and tag 6+2 (212 KB and 85 KB).
template <class P>
__host__ __device__ constexpr bool critic_built() { return MlpBuilt<P>::value && critic_smem_warps<P>(1) >= 1; }
// The compile-time cap of the two critic kernels, sized for one shared critic: MAPPO's register rule for its form
// (mlp_register_warps) unless an exception below holds (ptxas -v: no spills and no stack), lowered to what the shared
// critic's weights leave in shared memory.  The launcher lowers it at run time to critic_smem_warps(count).
// Forms by MAPPO's bits (kFormM: one episode, kFormME: episodes); the stack ptxas -v showed without the exception.
template <class P> struct CriticRegisterException : MlpException<0, 0> {};
template <> struct CriticRegisterException<Simple<1, 1>> : MlpException<kFormM, 12> {};                 // 8 at 128
template <> struct CriticRegisterException<Push<1, 1, 2>> : MlpException<kFormM | kFormME, 12> {};      // 32, 24 at 128
template <> struct CriticRegisterException<Crypto> : MlpException<kFormME, 12> {};                      // 24 at 128
template <> struct CriticRegisterException<Spread<4>> : MlpException<kFormM | kFormME, 8> {};           // 40, 40 at 168
template <> struct CriticRegisterException<Adversary<1, 3, 3>> : MlpException<kFormM | kFormME, 8> {};  // 8, 32 at 168
template <class P, bool EPISODES>
__host__ __device__ constexpr int critic_block_warps() {
    using X = CriticRegisterException<P>;
    constexpr int r = (X::forms >> (EPISODES ? 5 : 4) & 1) ? X::warps : mlp_register_warps<P, 64, EPISODES ? 5 : 4>();
    constexpr int s = critic_smem_warps<P>(1);
    return r < s ? r : s;
}
// one critic takes 21-60 KB where it is built (spread N=3: 37 KB); n per-agent ones fit next to the actor for simple,
// spread N=2 and 3, tag 1+1 and 2+1, adversary 1+2, push, speaker_listener, reference and crypto
static_assert(CriticShape<Simple<1, 1>>::kFloats * 4 == 21024 && CriticShape<Spread<5>>::kFloats * 4 == 59936,
              "simple: a 21 024 B critic; spread N=5: 59 936 B");
static_assert(CriticShape<Spread<3>>::kFloats * 4 == 37408 && critic_smem_warps<Spread<3>>(1) == 34 &&
              critic_smem_warps<Spread<3>>(3) == 12, "spread N=3: 75 360 + 37 408 + 34 x 3456 B; 3 critics, 12 warps");
static_assert(critic_smem_warps<Spread<5>>(1) == 7 && critic_smem_warps<Tag<4, 2, 2>>(1) == 6,
              "the smallest shared-critic blocks: spread N=5 7 warps, tag 4+2 6");
static_assert(critic_smem_warps<SpeakerListener>(2) == 53 && critic_smem_warps<Reference>(2) == 23 &&
              critic_smem_warps<Crypto>(3) == 38 && critic_smem_warps<Adversary<1, 2, 2>>(3) == 31,
              "per-agent critics that fit");
static_assert(critic_smem_warps<Adversary<1, 3, 3>>(4) < 1 && critic_smem_warps<Tag<3, 1, 2>>(4) < 1 &&
              critic_smem_warps<Spread<4>>(4) < 1 && critic_smem_warps<Spread<5>>(5) < 1 &&
              critic_smem_warps<Tag<4, 2, 2>>(6) < 1, "per-agent critics that do not fit");
static_assert(!critic_built<Spread<6>>() && !critic_built<Tag<6, 2, 3>>() && critic_built<Tag<4, 2, 2>>(),
              "no critic kernel for spread N=6 and tag 6+2");

// IPPO's local critics (MAPPO with use_centralized_V = False, next to MAPPO's actor, MlpCriticArgs): agent k's critic is
// the critic above on obs_k alone (share_obs = obs), laid out as CriticShape<P, k>.  count = 1: one shared critic, which
// needs every obs_dim_i equal, evaluated once per agent on that agent's observation; count = A: critic k evaluates agent
// k's, the sets back to back (LocalCriticShape::critic_off).  Agent k's values go to row k of values and final_values.
template <class P>
struct LocalCriticShape {
    __host__ __device__ static constexpr int floats(int k) {   // CriticShape<P, k>::kFloats for a run-time k
        return 64 * MlpShape<P, 64>::kt1(k) * 8 + 64 * 8 * 8 + 64 * 8 + 64 + 64 + 8;
    }
    __host__ __device__ static constexpr int critic_off(int k) { int s = 0; for (int j = 0; j < k; ++j) s += floats(j); return s; }
    __host__ __device__ static constexpr bool shared_ok() {
        for (int i = 1; i < P::A; ++i)
            if (P::obs_dim(i) != P::obs_dim(0)) return false;
        return true;
    }
    // the weights of `count` critics (1 or A)
    __host__ __device__ static constexpr int weight_floats(int count) { return count == 1 ? floats(0) : critic_off(P::A); }
    // the smallest set a call may pass: one shared critic where the agents observe alike, else A
    static constexpr int kMinFloats = weight_floats(shared_ok() ? 1 : P::A);
};
template <class P>
__host__ __device__ constexpr int local_critic_smem_warps(int count) {
    return (kMlpSmemBytes / 4 - MlpShape<P, 64>::kWeightFloats - LocalCriticShape<P>::weight_floats(count)) /
           MlpShape<P, 64>::kWarpFloats;
}
// Built where the smallest set leaves room for a warp: every MAPPO program but tag 4+2 (per-agent critics only, 150 720
// B of them with 81 728 B free) and tag 6+2 (15 104 B free next to its actor)
template <class P>
__host__ __device__ constexpr bool local_critic_built() {
    return MlpBuilt<P>::value && local_critic_smem_warps<P>(LocalCriticShape<P>::shared_ok() ? 1 : P::A) >= 1;
}
// The compile-time cap of the two local-critic kernels: MAPPO's register rule for its form unless an exception below
// holds (ptxas -v: no spills and no stack), lowered to what the smallest set leaves in shared memory.  The launcher
// lowers it at run time to local_critic_smem_warps(count).  Forms by MAPPO's bits; the stack ptxas -v showed without
// the exception.
template <class P> struct LocalCriticRegisterException : MlpException<0, 0> {};
template <> struct LocalCriticRegisterException<Simple<1, 1>> : MlpException<kFormM, 12> {};                 // 16 at 128
template <> struct LocalCriticRegisterException<Push<1, 1, 2>> : MlpException<kFormM | kFormME, 12> {};      // 40, 48 at 128
template <> struct LocalCriticRegisterException<Crypto> : MlpException<kFormME, 12> {};                      // 56 at 128
template <> struct LocalCriticRegisterException<Reference> : MlpException<kFormME, 8> {};                    // 32 at 168
template <> struct LocalCriticRegisterException<Spread<4>> : MlpException<kFormM | kFormME, 8> {};           // 8, 8 at 168
template <> struct LocalCriticRegisterException<Spread<5>> : MlpException<kFormM, 8> {};                     // 8 at 168
template <> struct LocalCriticRegisterException<Adversary<1, 3, 3>> : MlpException<kFormM | kFormME, 8> {};  // 16, 8 at 168
template <class P, bool EPISODES>
__host__ __device__ constexpr int local_critic_block_warps() {
    using X = LocalCriticRegisterException<P>;
    constexpr int r = (X::forms >> (EPISODES ? 5 : 4) & 1) ? X::warps : mlp_register_warps<P, 64, EPISODES ? 5 : 4>();
    constexpr int s = local_critic_smem_warps<P>(LocalCriticShape<P>::shared_ok() ? 1 : P::A);
    return r < s ? r : s;
}
static_assert(LocalCriticShape<Spread<3>>::floats(0) * 4 == 25120 && local_critic_smem_warps<Spread<3>>(3) == 23,
              "spread N=3: 3 x 25 120 B of critics next to 75 360 B of actor, 23 warps");
static_assert(LocalCriticShape<Spread<6>>::floats(0) * 4 == 29216 && local_critic_smem_warps<Spread<6>>(1) == 4 &&
              local_critic_smem_warps<Spread<6>>(6) < 1, "spread N=6: one shared 29 216 B critic, 4 warps");
static_assert(local_critic_smem_warps<Spread<5>>(1) >= 1 && local_critic_smem_warps<Spread<5>>(5) < 1,
              "spread N=5: a shared critic fits, five do not");
static_assert(kMlpSmemBytes - MlpShape<Tag<6, 2, 3>, 64>::kWeightFloats * 4 == 15104 && !local_critic_built<Tag<6, 2, 3>>(),
              "tag 6+2: 15 104 B free, no local critic");

// rMAPPO's recurrent centralized critic (R_Critic with use_recurrent_policy, recurrent_N = 1, use_centralized_V), one
// weight set shared by every agent, in a kernel of its own that runs after the recurrent actor's rollout and reads its
// observation records:
//     x = MLPBase(share_obs) = [LN(D)] -> Linear(D, 64) -> act -> LN(64) -> Linear(64, 64) -> act -> LN(64)
//     h' = GRU(x, h),  V = Linear(64, 1)(LN(h'))
// folded as the recurrent actor is (the base's last LayerNorm into w_ih, b_ih; the GRU's LayerNorm into w3, b3).
// share_obs is every agent's raw observation in agent order (D = sum of obs_dim_i), read from obs[i] ([T][n][obs_dim_i])
// at step t and from final_obs[i] ([E][n][obs_dim_i]) for the bootstrap value.  Every L steps (L = 0: one episode of T)
// the episode ends: its bootstrap value V(final_obs[e], h') goes to final_values[e] and h restarts from 0.  With L = 0,
// h starts from h [n][64] (read); h receives the h after the last step in both forms, h_rec ([T][n][64] or null) the h
// each step's critic consumed.  values [T][A][n] and final_values [E][A][n] hold the shared value for every agent.
struct RCriticArgs {
    const float *obs[kMaxA], *final_obs[kMaxA];
    const float *w1, *b1, *w2, *b2, *w_ih, *b_ih, *w_hh, *b_hh, *w3, *b3;
    float *h, *h_rec, *values, *final_values;
    int64_t n;
    int32_t T, L;
    uint32_t net_flags;
    float ln_eps;
};
static_assert(sizeof(RCriticArgs) <= 4096, "kernel parameter space");
// rMAPPO's per-agent recurrent critics (the separated runner: agent k's own R_Critic on share_obs), one launch with
// blockIdx.y = k: c as above but for the weights, which are w[j][k] (W1, b1, W2, b2, W_ih, b_ih, W_hh, b_hh, W3, b3),
// and critic k's state, h [A][n][64] and h_rec [T][A][n][64] (or null), its slice k; critic k writes only agent k's row
// of values and final_values.
struct RCriticSeparatedArgs {
    RCriticArgs c;
    const float *w[10][kMaxA];
};
static_assert(sizeof(RCriticSeparatedArgs) <= 4096, "kernel parameter space");

// Its weights in shared memory, in floats: W1's B fragments agent by agent as the MLP critic's (CriticShape::w1_off,
// stage_critic_w1), then W2, W_ih and W_hh (GruShape's layout), W3 (one n-tile, its one real column first), b1 [64],
// b2 [64], b_ih [192], b_hh [192], b3 [8]: 512 sum(kt1_i) + 29 704 floats.  The records stream through registers (no
// per-warp tile), so the rest of shared memory is the L1 cache that serves their second and third reads.  K >= 0: the
// local critic of IPPO on agent K's observation alone (CriticShape<P, K>'s W1), 512 kt1_K + 29 704 floats.
template <class P, int K = -1>
struct RCriticShape {
    using C = CriticShape<P, K>;
    static constexpr int NT = 8, NG = 24;
    static constexpr int w2_off = C::w2_off;
    static constexpr int wih_off = w2_off + 64 * NT * NT;
    static constexpr int whh_off = wih_off + 64 * NT * NG;
    static constexpr int w3_off = whh_off + 64 * NT * NG;
    static constexpr int b1_off = w3_off + 64 * NT;
    static constexpr int b2_off = b1_off + 64;
    static constexpr int bih_off = b2_off + 64;
    static constexpr int bhh_off = bih_off + 192;
    static constexpr int b3_off = bhh_off + 192;
    static constexpr int kFloats = b3_off + 8;
};
static_assert(RCriticShape<Simple<1, 1>>::kFloats * 4 == 120864 && RCriticShape<Spread<3>>::kFloats * 4 == 137248 &&
              RCriticShape<Reference>::kFloats * 4 == 131104 && RCriticShape<Spread<6>>::kFloats * 4 == 180256,
              "simple 120 864 B, spread N=3 137 248 B, simple_reference 131 104 B, spread N=6 180 256 B");
static_assert(RCriticShape<Spread<6>>::kFloats * 4 <= kMlpSmemBytes, "the largest weight set fits an SM");
// Warps per block, every program: 8 (255 registers per thread for h, its TF32 copy, x and the gate accumulators of
// one m-tile; ptxas -v: no spills, no stack).  Each warp owns 16 worlds; one block per SM.
constexpr int kRCriticWarps = 8;

__device__ __forceinline__ uint32_t to_tf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}
// d += a . b, one m16n8k8 TF32 tile (A row-major 16 x 8, B column-major 8 x 8, fp32 accumulators)
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], float2 b) {
    asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(__float_as_uint(b.x)), "r"(__float_as_uint(b.y)));
}

// W ([NV][KV], torch Linear layout, global) -> TF32 B fragments in shared memory, [KT][NTT][lane][2], zero outside
// [NV][KV].  Fragment element j of lane l in tile (kt, nt) is B[k][n] = W[n][k] with n = nt*8 + l/4 and
// k = kt*8 + l%4 + 4j (PERM = false: A comes from the observation tile) or k = kt*8 + 2(l%4) + j (PERM = true: A is the
// previous layer's accumulator fragment).  Consecutive lanes read consecutive float2: conflict-free LDS.64.
template <int KT, int NTT, bool PERM>
__device__ __forceinline__ void stage_fragments(float *dst, const float *__restrict__ W, int NV, int KV) {
    for (int q = threadIdx.x; q < KT * NTT * 64; q += blockDim.x) {
        const int j = q & 1, l = (q >> 1) & 31, tile = q >> 6;
        const int nt = tile % NTT, kt = tile / NTT;
        const int nn = nt * 8 + (l >> 2);
        const int k = kt * 8 + (PERM ? 2 * (l & 3) + j : (l & 3) + 4 * j);
        dst[q] = __uint_as_float(to_tf32((nn < NV && k < KV) ? W[nn * KV + k] : 0.0f));
    }
}

// accumulator fragment -> ReLU -> TF32 A fragment of the next layer (k order permuted as in stage_fragments)
__device__ __forceinline__ void relu_tf32_frag(uint32_t (&a)[4], const float (&c)[4]) {
    a[0] = to_tf32(fmaxf(c[0], 0.0f));   // row g,   k = 2q
    a[1] = to_tf32(fmaxf(c[2], 0.0f));   // row g+8, k = 2q
    a[2] = to_tf32(fmaxf(c[1], 0.0f));   // row g,   k = 2q+1
    a[3] = to_tf32(fmaxf(c[3], 0.0f));   // row g+8, k = 2q+1
}

// MAPPO's hidden layer: the accumulators of one m-tile (NT n-tiles) -> act (tanhf, or ReLU) -> LayerNorm without affine
// -> TF32 A fragments of the next layer, in relu_tf32_frag's order.  A row's NT * 8 units are 2 per n-tile in each of
// the 4 lanes of a quad (rows g: elements 0, 1; g + 8: 2, 3), so its sums are a local sum and __shfl_xor over 1 and 2.
// Two-pass fp32 statistics as torch takes them: mu = sum(x) / H, then var = sum((x - mu)^2) / H; the normalised value
// (x - mu) * rsqrt(var + eps) is rounded to TF32 only then.
// The LayerNorm alone (norm_tf32_frags) also normalises the recurrent actor's h'.
template <int NT>
__device__ __forceinline__ void norm_tf32_frags(uint32_t (&a)[NT][4], const float (&c)[NT][4], float eps);
template <int NT>
__device__ __forceinline__ void act_norm_tf32_frags(uint32_t (&a)[NT][4], float (&c)[NT][4], bool tanh_act, float eps) {
    if (tanh_act) {
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
#pragma unroll
            for (int j = 0; j < 4; ++j) c[nt][j] = tanhf(c[nt][j]);
    } else {
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
#pragma unroll
            for (int j = 0; j < 4; ++j) c[nt][j] = fmaxf(c[nt][j], 0.0f);
    }
    norm_tf32_frags<NT>(a, c, eps);
}
template <int NT>
__device__ __forceinline__ void norm_tf32_frags(uint32_t (&a)[NT][4], const float (&c)[NT][4], float eps) {
    constexpr float kInvH = 1.0f / (NT * 8);      // H = 8 NT, a power of two: exact
    float s0 = 0.0f, s1 = 0.0f;
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) { s0 += c[nt][0] + c[nt][1]; s1 += c[nt][2] + c[nt][3]; }
    s0 += __shfl_xor_sync(0xffffffffu, s0, 1); s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
    s0 += __shfl_xor_sync(0xffffffffu, s0, 2); s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
    const float m0 = s0 * kInvH, m1 = s1 * kInvH;
    float v0 = 0.0f, v1 = 0.0f;
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
        const float d0 = c[nt][0] - m0, d1 = c[nt][1] - m0, d2 = c[nt][2] - m1, d3 = c[nt][3] - m1;
        v0 += d0 * d0 + d1 * d1;
        v1 += d2 * d2 + d3 * d3;
    }
    v0 += __shfl_xor_sync(0xffffffffu, v0, 1); v1 += __shfl_xor_sync(0xffffffffu, v1, 1);
    v0 += __shfl_xor_sync(0xffffffffu, v0, 2); v1 += __shfl_xor_sync(0xffffffffu, v1, 2);
    const float r0 = rsqrtf(v0 * kInvH + eps), r1 = rsqrtf(v1 * kInvH + eps);
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
        a[nt][0] = to_tf32((c[nt][0] - m0) * r0);   // row g,   k = 2q
        a[nt][1] = to_tf32((c[nt][2] - m1) * r1);   // row g+8, k = 2q
        a[nt][2] = to_tf32((c[nt][1] - m0) * r0);   // row g,   k = 2q+1
        a[nt][3] = to_tf32((c[nt][3] - m1) * r1);   // row g+8, k = 2q+1
    }
}

// One GRU step of one m-tile, hidden width 64, torch's gate order r, z, n (GruShape's layout: W_ih's and W_hh's B
// fragments [k-tile][24 n-tiles][lane][2], b_ih and b_hh [192]):
//     r = sigmoid(W_ir x + b_ir + W_hr h + b_hr),  z = sigmoid(W_iz x + b_iz + W_hz h + b_hz)
//     n = tanh(W_in x + b_in + r * (W_hn h + b_hn)),  h' = (1 - z) * n + z * h
// x and ht are the TF32 A fragments of x and h, hn receives h' in the accumulator layout.  For units j * 8 .. j * 8 + 7
// r and z each accumulate both GEMMs and both biases, n keeps W_in x + b_in and W_hn h + b_hn apart; h_of(j, hf) then
// supplies the unrounded h of those units (elements as the accumulators').  expf and tanhf are full precision.  The
// recurrent critic's cell; mlp_agent's GRU branch computes the same operations in the same order inline (calling this
// from there changed the recurrent actor's SASS).
template <class HOf>
__device__ __forceinline__ void gru_cell(const float *Wih, const float *Whh, const float *Bih, const float *Bhh,
                                         const uint32_t (&x)[8][4], const uint32_t (&ht)[8][4], int lane, float (&hn)[8][4],
                                         HOf &&h_of) {
    constexpr int NT = 8, NG = 24;
    const int tq = lane & 3;
#pragma unroll
    for (int j = 0; j < NT; ++j) {
        float r[4], z[4], ni[4], nh[4];
        {
            const float2 bir = *reinterpret_cast<const float2 *>(Bih + j * 8 + 2 * tq);
            const float2 bhr = *reinterpret_cast<const float2 *>(Bhh + j * 8 + 2 * tq);
            const float2 biz = *reinterpret_cast<const float2 *>(Bih + 64 + j * 8 + 2 * tq);
            const float2 bhz = *reinterpret_cast<const float2 *>(Bhh + 64 + j * 8 + 2 * tq);
            const float2 bin = *reinterpret_cast<const float2 *>(Bih + 128 + j * 8 + 2 * tq);
            const float2 bhn = *reinterpret_cast<const float2 *>(Bhh + 128 + j * 8 + 2 * tq);
            r[0] = r[2] = bir.x + bhr.x; r[1] = r[3] = bir.y + bhr.y;
            z[0] = z[2] = biz.x + bhz.x; z[1] = z[3] = biz.y + bhz.y;
            ni[0] = ni[2] = bin.x; ni[1] = ni[3] = bin.y;
            nh[0] = nh[2] = bhn.x; nh[1] = nh[3] = bhn.y;
        }
#pragma unroll
        for (int kt = 0; kt < NT; ++kt) {
            const float *bi = Wih + ((kt * NG + j) * 32 + lane) * 2, *bh = Whh + ((kt * NG + j) * 32 + lane) * 2;
            mma_tf32(r, x[kt], *reinterpret_cast<const float2 *>(bi));
            mma_tf32(r, ht[kt], *reinterpret_cast<const float2 *>(bh));
            mma_tf32(z, x[kt], *reinterpret_cast<const float2 *>(bi + NT * 64));
            mma_tf32(z, ht[kt], *reinterpret_cast<const float2 *>(bh + NT * 64));
            mma_tf32(ni, x[kt], *reinterpret_cast<const float2 *>(bi + 2 * NT * 64));
            mma_tf32(nh, ht[kt], *reinterpret_cast<const float2 *>(bh + 2 * NT * 64));
        }
        float hf[4];
        h_of(j, hf);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float rg = 1.0f / (1.0f + expf(-r[e])), zg = 1.0f / (1.0f + expf(-z[e]));
            const float ng = tanhf(ni[e] + rg * nh[e]);
            hn[j][e] = (1.0f - zg) * ng + zg * hf[e];
        }
    }
}

// pr[B, B + K) = softmax(z[B, B + K)): one action sub-space.  The operation order is the one of every other softmax
// here (the max is exact in any order; the sum runs from the first entry to the last).
template <int B, int K, int N>
__device__ __forceinline__ void softmax_segment(const float (&z)[N], float (&pr)[N]) {
    static_assert(B + K <= N, "segment inside the action vector");
    float m = z[B];
#pragma unroll
    for (int c = 1; c < K; ++c) m = fmaxf(m, z[B + c]);
    float e[K], sum = 0.0f;
#pragma unroll
    for (int c = 0; c < K; ++c) { e[c] = expf(__fsub_rn(z[B + c], m)); sum = __fadd_rn(sum, e[c]); }
#pragma unroll
    for (int c = 0; c < K; ++c) pr[B + c] = __fdiv_rn(e[c], sum);
}

// One sub-space of the categorical form: pr[B, B + K) = one_hot(k), k = argmax zs[B, B + K) with the lowest index
// winning ties (zs: the perturbed logits when exploring, else z), and the return value log_softmax(z[B, B + K))[k] of
// the unperturbed logits, its max and sum formed as in softmax_segment.  k is selected, never used as an index, so
// the arrays stay in registers.
template <int B, int K, int N>
__device__ __forceinline__ float categorical_segment(const float (&zs)[N], const float (&z)[N], float (&pr)[N], int &k) {
    static_assert(B + K <= N, "segment inside the action vector");
    float best = zs[B], zk = z[B], m = z[B];
    k = 0;
#pragma unroll
    for (int c = 1; c < K; ++c) {
        if (zs[B + c] > best) { best = zs[B + c]; zk = z[B + c]; k = c; }
        m = fmaxf(m, z[B + c]);
    }
    float sum = 0.0f;
#pragma unroll
    for (int c = 0; c < K; ++c) sum = __fadd_rn(sum, expf(__fsub_rn(z[B + c], m)));
#pragma unroll
    for (int c = 0; c < K; ++c) pr[B + c] = c == k ? 1.0f : 0.0f;
    return __fsub_rn(__fsub_rn(zk, m), logf(sum));
}

// one agent of the tensor-core actor for the warp's 32 worlds: observation -> tile -> 3 GEMMs -> this lane's logits ->
// (Gumbel-)softmax per sub-space -> decoded (u.x, u.y), and a speaker's utterance into cact[I * dim_c ...].  Called by
// all 32 lanes (mma.sync is warp-collective).  t indexes the records.  The exploration noise is keyed by (pa.epoch, t),
// and in the episode form (EPISODES) by (epoch, step) = (pa.epoch + e, t - e * T) in episode e.  The categorical form
// (CATEGORICAL) applies one-hot vectors instead of the softmax and writes the records of cr.  MAPPO evaluates MAPPO's
// actor (MlpMappoArgs) with the same GEMMs: after the observation record, the input LayerNorm (net_flags &
// kMappoFeatureNorm) normalises each lane's tile row in place; act_norm_tf32_frags replaces relu_tf32_frag; and since
// the second LayerNorm needs a whole row of h2, layers 2 and 3 run one m-tile at a time (h2 of 16 rows in 32 fp32
// registers, W2's B fragments read once per m-tile).
// GRU adds MAPPO's recurrent actor (MlpGruArgs) to MAPPO's: per m-tile the base's two layers, the GRU step, the
// LayerNorm of h' and the head, so that x, h and h' fit in registers.  The weights are agent I's set in
// GruAgentShape<P, I>'s layout: the one shared set (GruShape), or the slot the separated actor restages for agent I.
//
// Where the base's second layer, the head and their biases sit in Wsm: the agent's block (MlpShape), or the GRU set
template <class P, int H, int I, bool GRU>
struct AgentWeights {
    using S = MlpShape<P, H>;
    static constexpr int w2 = S::w2_off(I), w3 = S::w3_off(I), b1 = S::b1_off(I), b2 = S::b2_off(I), b3 = S::b3_off(I);
};
template <class P, int I>
struct AgentWeights<P, 64, I, true> {
    using G = GruAgentShape<P, I>;
    static constexpr int w2 = G::w2_off, w3 = G::w3_off, b1 = G::b1_off, b2 = G::b2_off, b3 = G::b3_off;
};
template <class P, int H, int I, bool EPISODES = false, bool CATEGORICAL = false, bool MAPPO = false, bool GRU = false>
__device__ __forceinline__ float2 mlp_agent(const MlpPolicyArgs &pa, const typename P::W &w, const float *__restrict__ Wsm,
                                            float *s_warp, int lane, int t, int rows, bool active, int64_t w0, int64_t wi,
                                            float *cact, int step = 0, uint64_t epoch = 0,
                                            const MlpCategoricalRecords *cr = nullptr, float ln_eps = 0.0f,
                                            uint32_t net_flags = 0, const MlpGruState *gs = nullptr) {
    static_assert(!MAPPO || (CATEGORICAL && H == 64), "the MAPPO actor: categorical form, H = 64");
    static_assert(!GRU || MAPPO, "the recurrent actor is MAPPO's");
    using S = MlpShape<P, H>;
    using O = AgentWeights<P, H, I, GRU>;
    constexpr int OD = P::obs_dim(I), KT1 = S::kt1(I), NT = S::NT, PITCH = ObsTile<OD>::kPitch;
    constexpr int AD = P::act_dim(I), NO = S::nout(I) / 8;
    constexpr int MOVE = P::movable(I) ? 5 : 0, COMM = I < P::NS ? P::DIMC : 0;   // sub-spaces, speakers come first
    static_assert(MOVE + COMM == AD && AD > 0, "action vector = [movement][utterance]");
    const DevDesc &d = pa.s.d;
    const int64_t n = pa.s.n;
    float *tile = s_warp;
    float *lgs = s_warp + S::kLogitOff;
    {
        TileWriter<OD> o(tile, lane);
        P::template observe<I>(d, w, o);                   // scenario.observation(agent I) -> this lane's tile row
    }
    __syncwarp();
    if (pa.obs_rec[I] != nullptr)                          // the observation the actor sees at step t
        store_obs_rows<OD>(pa.obs_rec[I] + (static_cast<int64_t>(t) * n + w0) * OD, tile, lane, rows, active);
    if constexpr (MAPPO) {
        if (net_flags & kMappoFeatureNorm) {               // the record holds the raw observation; the actor sees it normalised
            __syncwarp();                                  // every lane has streamed the tile
            float *row = tile + lane * PITCH;              // odd pitch: conflict-free
            float s = 0.0f;
#pragma unroll
            for (int c = 0; c < OD; ++c) s += row[c];
            const float mu = s / static_cast<float>(OD);
            float v = 0.0f;
#pragma unroll
            for (int c = 0; c < OD; ++c) { const float dc = row[c] - mu; v += dc * dc; }
            const float rstd = rsqrtf(v / static_cast<float>(OD) + ln_eps);
#pragma unroll
            for (int c = 0; c < OD; ++c) row[c] = (row[c] - mu) * rstd;
            __syncwarp();
        }
    }
    const int gq = lane >> 2, tq = lane & 3;
    // ---- layer 1: [32 x K1] . [K1 x H] + b1 ----
    float h[2][NT][4];
    const float *B1 = Wsm + O::b1;
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
        const float2 b = *reinterpret_cast<const float2 *>(B1 + nt * 8 + 2 * tq);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) { h[mt][nt][0] = b.x; h[mt][nt][1] = b.y; h[mt][nt][2] = b.x; h[mt][nt][3] = b.y; }
    }
#pragma unroll
    for (int kt = 0; kt < KT1; ++kt) {
        uint32_t a[2][4];
        const int c0 = kt * 8 + tq, c1 = c0 + 4;
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
            const float *r0 = tile + (mt * 16 + gq) * PITCH, *r1 = r0 + 8 * PITCH;
            if (kt * 8 + 8 <= OD) {
                a[mt][0] = to_tf32(r0[c0]); a[mt][1] = to_tf32(r1[c0]);
                a[mt][2] = to_tf32(r0[c1]); a[mt][3] = to_tf32(r1[c1]);
            } else {                                       // columns >= obs_dim are the zero padding of K1
                a[mt][0] = to_tf32(c0 < OD ? r0[c0] : 0.0f); a[mt][1] = to_tf32(c0 < OD ? r1[c0] : 0.0f);
                a[mt][2] = to_tf32(c1 < OD ? r0[c1] : 0.0f); a[mt][3] = to_tf32(c1 < OD ? r1[c1] : 0.0f);
            }
        }
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            const float2 b = *reinterpret_cast<const float2 *>(Wsm + ((kt * NT + nt) * 32 + lane) * 2);
            mma_tf32(h[0][nt], a[0], b);
            mma_tf32(h[1][nt], a[1], b);
        }
    }
    uint32_t x1[2][NT][4];
    if constexpr (GRU) {
        // the recurrent actor runs layer 1 again one m-tile at a time (below): h above is dead code for it
    } else if constexpr (MAPPO) {
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) act_norm_tf32_frags<NT>(x1[mt], h[mt], net_flags & kMappoTanh, ln_eps);
    } else {
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) relu_tf32_frag(x1[mt][nt], h[mt][nt]);
    }
    // ---- layers 2 and 3, one 8-unit tile of h2 at a time: logits += relu(x1 . W2^T[:, tile] + b2[tile]) . W3^T[tile, :]
    const float *W2 = Wsm + O::w2, *W3 = Wsm + O::w3, *B2 = Wsm + O::b2, *B3 = Wsm + O::b3;
    float lg[2][NO][4];
#pragma unroll
    for (int ot = 0; ot < NO; ++ot) {
        const float2 b = *reinterpret_cast<const float2 *>(B3 + ot * 8 + 2 * tq);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) { lg[mt][ot][0] = b.x; lg[mt][ot][1] = b.y; lg[mt][ot][2] = b.x; lg[mt][ot][3] = b.y; }
    }
    if constexpr (GRU) {   // ---- the recurrent actor, one m-tile (16 worlds) at a time: layers 1 and 2 with their
                           //      LayerNorms -> x, h' = GRU(x, h), logits += LN(h') . W3^T
        using G = GruAgentShape<P, I>;
        const float *Wih = Wsm + G::wih_off, *Whh = Wsm + G::whh_off, *Bih = Wsm + G::bih_off, *Bhh = Wsm + G::bhh_off;
        const bool h_zero = EPISODES && step == 0;         // every episode starts from h = 0
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
            uint32_t x[NT][4];
            {
                float c[NT][4];
#pragma unroll
                for (int nt = 0; nt < NT; ++nt) {
                    const float2 b = *reinterpret_cast<const float2 *>(B1 + nt * 8 + 2 * tq);
                    c[nt][0] = b.x; c[nt][1] = b.y; c[nt][2] = b.x; c[nt][3] = b.y;
                }
#pragma unroll
                for (int kt = 0; kt < KT1; ++kt) {
                    uint32_t a[4];
                    const int c0 = kt * 8 + tq, c1 = c0 + 4;
                    const float *r0 = tile + (mt * 16 + gq) * PITCH, *r1 = r0 + 8 * PITCH;
                    a[0] = to_tf32(c0 < OD ? r0[c0] : 0.0f); a[1] = to_tf32(c0 < OD ? r1[c0] : 0.0f);
                    a[2] = to_tf32(c1 < OD ? r0[c1] : 0.0f); a[3] = to_tf32(c1 < OD ? r1[c1] : 0.0f);
#pragma unroll
                    for (int nt = 0; nt < NT; ++nt)
                        mma_tf32(c[nt], a, *reinterpret_cast<const float2 *>(Wsm + ((kt * NT + nt) * 32 + lane) * 2));
                }
                uint32_t xa[NT][4];
                act_norm_tf32_frags<NT>(xa, c, net_flags & kMappoTanh, ln_eps);
#pragma unroll
                for (int nt = 0; nt < NT; ++nt) {
                    const float2 bb = *reinterpret_cast<const float2 *>(B2 + nt * 8 + 2 * tq);
                    c[nt][0] = bb.x; c[nt][1] = bb.y; c[nt][2] = bb.x; c[nt][3] = bb.y;
#pragma unroll
                    for (int kt = 0; kt < NT; ++kt)
                        mma_tf32(c[nt], xa[kt], *reinterpret_cast<const float2 *>(W2 + ((kt * NT + nt) * 32 + lane) * 2));
                }
                act_norm_tf32_frags<NT>(x, c, net_flags & kMappoTanh, ln_eps);
            }
            // this lane's rows g and g + 8 of the m-tile in the accumulator layout (units nt * 8 + 2 tq, + 1): a quad
            // reads and writes whole 32-byte sectors.  Idle rows replay world w0 and store nothing.
            const int ra = mt * 16 + gq, rb = ra + 8;
            const int64_t wa = w0 + (ra < rows ? ra : 0), wb = w0 + (rb < rows ? rb : 0);
            float *ha = gs->h + (static_cast<int64_t>(I) * n + wa) * 64 + 2 * tq;
            float *hb = gs->h + (static_cast<int64_t>(I) * n + wb) * 64 + 2 * tq;
            // h as W_hh's A operand, TF32: the accumulator layout is relu_tf32_frag's permuted A layout
            uint32_t ht[NT][4];
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) {
                const float2 va = h_zero ? make_float2(0.0f, 0.0f) : *reinterpret_cast<const float2 *>(ha + nt * 8);
                const float2 vb = h_zero ? make_float2(0.0f, 0.0f) : *reinterpret_cast<const float2 *>(hb + nt * 8);
                if (gs->h_rec != nullptr) {                // the h this step's actor consumes
                    float *qa = gs->h_rec + ((static_cast<int64_t>(t) * P::A + I) * n + wa) * 64 + 2 * tq;
                    float *qb = gs->h_rec + ((static_cast<int64_t>(t) * P::A + I) * n + wb) * 64 + 2 * tq;
                    if (ra < rows) *reinterpret_cast<float2 *>(qa + nt * 8) = va;
                    if (rb < rows) *reinterpret_cast<float2 *>(qb + nt * 8) = vb;
                }
                ht[nt][0] = to_tf32(va.x); ht[nt][1] = to_tf32(vb.x); ht[nt][2] = to_tf32(va.y); ht[nt][3] = to_tf32(vb.y);
            }
            // h' for units j * 8 .. j * 8 + 7: r and z each accumulate both GEMMs and both biases, n keeps W_in x + b_in
            // and W_hn h + b_hn apart.  The update reads the unrounded h of those units again (L1) rather than holding
            // all of it next to its TF32 copy.
            float hn[NT][4];
#pragma unroll
            for (int j = 0; j < NT; ++j) {
                float r[4], z[4], ni[4], nh[4];
                {
                    const float2 bir = *reinterpret_cast<const float2 *>(Bih + j * 8 + 2 * tq);
                    const float2 bhr = *reinterpret_cast<const float2 *>(Bhh + j * 8 + 2 * tq);
                    const float2 biz = *reinterpret_cast<const float2 *>(Bih + 64 + j * 8 + 2 * tq);
                    const float2 bhz = *reinterpret_cast<const float2 *>(Bhh + 64 + j * 8 + 2 * tq);
                    const float2 bin = *reinterpret_cast<const float2 *>(Bih + 128 + j * 8 + 2 * tq);
                    const float2 bhn = *reinterpret_cast<const float2 *>(Bhh + 128 + j * 8 + 2 * tq);
                    r[0] = r[2] = bir.x + bhr.x; r[1] = r[3] = bir.y + bhr.y;
                    z[0] = z[2] = biz.x + bhz.x; z[1] = z[3] = biz.y + bhz.y;
                    ni[0] = ni[2] = bin.x; ni[1] = ni[3] = bin.y;
                    nh[0] = nh[2] = bhn.x; nh[1] = nh[3] = bhn.y;
                }
#pragma unroll
                for (int kt = 0; kt < NT; ++kt) {
                    const float *bi = Wih + ((kt * G::NG + j) * 32 + lane) * 2, *bh = Whh + ((kt * G::NG + j) * 32 + lane) * 2;
                    mma_tf32(r, x[kt], *reinterpret_cast<const float2 *>(bi));
                    mma_tf32(r, ht[kt], *reinterpret_cast<const float2 *>(bh));
                    mma_tf32(z, x[kt], *reinterpret_cast<const float2 *>(bi + NT * 64));
                    mma_tf32(z, ht[kt], *reinterpret_cast<const float2 *>(bh + NT * 64));
                    mma_tf32(ni, x[kt], *reinterpret_cast<const float2 *>(bi + 2 * NT * 64));
                    mma_tf32(nh, ht[kt], *reinterpret_cast<const float2 *>(bh + 2 * NT * 64));
                }
                const float2 va = h_zero ? make_float2(0.0f, 0.0f) : *reinterpret_cast<const float2 *>(ha + j * 8);
                const float2 vb = h_zero ? make_float2(0.0f, 0.0f) : *reinterpret_cast<const float2 *>(hb + j * 8);
                const float hf[4] = {va.x, va.y, vb.x, vb.y};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float rg = 1.0f / (1.0f + expf(-r[e])), zg = 1.0f / (1.0f + expf(-z[e]));
                    const float ng = tanhf(ni[e] + rg * nh[e]);
                    hn[j][e] = (1.0f - zg) * ng + zg * hf[e];
                }
            }
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) {
                if (ra < rows) *reinterpret_cast<float2 *>(ha + nt * 8) = make_float2(hn[nt][0], hn[nt][1]);
                if (rb < rows) *reinterpret_cast<float2 *>(hb + nt * 8) = make_float2(hn[nt][2], hn[nt][3]);
            }
            uint32_t xh[NT][4];
            norm_tf32_frags<NT>(xh, hn, ln_eps);
#pragma unroll
            for (int ot = 0; ot < NO; ++ot)
#pragma unroll
                for (int kt = 0; kt < NT; ++kt)
                    mma_tf32(lg[mt][ot], xh[kt], *reinterpret_cast<const float2 *>(W3 + ((kt * NO + ot) * 32 + lane) * 2));
            __syncwarp();   // as in MAPPO's branch: the second m-tile reads its B fragments again
        }
    } else if constexpr (MAPPO) {   // ---- MAPPO: per m-tile, h2 = x1 . W2^T + b2 whole, act + LayerNorm, then logits += x2 . W3^T
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
            float c[NT][4];
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) {
                const float2 bb = *reinterpret_cast<const float2 *>(B2 + nt * 8 + 2 * tq);
                c[nt][0] = bb.x; c[nt][1] = bb.y; c[nt][2] = bb.x; c[nt][3] = bb.y;
#pragma unroll
                for (int kt = 0; kt < NT; ++kt)
                    mma_tf32(c[nt], x1[mt][kt], *reinterpret_cast<const float2 *>(W2 + ((kt * NT + nt) * 32 + lane) * 2));
            }
            uint32_t x2[NT][4];
            act_norm_tf32_frags<NT>(x2, c, net_flags & kMappoTanh, ln_eps);
#pragma unroll
            for (int ot = 0; ot < NO; ++ot)
#pragma unroll
                for (int kt = 0; kt < NT; ++kt)
                    mma_tf32(lg[mt][ot], x2[kt], *reinterpret_cast<const float2 *>(W3 + ((kt * NO + ot) * 32 + lane) * 2));
            // a memory barrier for the compiler: it would otherwise keep all of W2's and W3's B fragments (up to 160
            // registers) live from the first m-tile to the second instead of reading them again
            __syncwarp();
        }
    } else {
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
        float c[2][4];
        const float2 bb = *reinterpret_cast<const float2 *>(B2 + nt * 8 + 2 * tq);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) { c[mt][0] = bb.x; c[mt][1] = bb.y; c[mt][2] = bb.x; c[mt][3] = bb.y; }
#pragma unroll
        for (int kt = 0; kt < NT; ++kt) {
            const float2 b = *reinterpret_cast<const float2 *>(W2 + ((kt * NT + nt) * 32 + lane) * 2);
            mma_tf32(c[0], x1[0][kt], b);
            mma_tf32(c[1], x1[1][kt], b);
        }
#pragma unroll
        for (int ot = 0; ot < NO; ++ot) {
            const float2 b3 = *reinterpret_cast<const float2 *>(W3 + ((nt * NO + ot) * 32 + lane) * 2);
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
                uint32_t x2[4];
                relu_tf32_frag(x2, c[mt]);
                mma_tf32(lg[mt][ot], x2, b3);
            }
        }
    }
    }
    // ---- logits back to their lane (row r = world w0 + r) ----
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int ot = 0; ot < NO; ++ot) {
            float *r0 = lgs + (mt * 16 + gq) * S::kLogitPitch + ot * 8 + 2 * tq, *r1 = r0 + 8 * S::kLogitPitch;
            r0[0] = lg[mt][ot][0]; r0[1] = lg[mt][ot][1];
            r1[0] = lg[mt][ot][2]; r1[1] = lg[mt][ot][3];
        }
    __syncwarp();
    float z[AD];
#pragma unroll
    for (int c = 0; c < AD; ++c) z[c] = lgs[lane * S::kLogitPitch + c];
    float zl[CATEGORICAL ? AD : 1];                        // the unperturbed logits: the log-probability's
    if constexpr (CATEGORICAL) {
#pragma unroll
        for (int c = 0; c < AD; ++c) zl[c] = z[c];
    }
    if (pa.explore) {                                      // Gumbel-softmax sample (see the definition above)
        const uint64_t gw = pa.world_offset + static_cast<uint64_t>(wi);
        const uint2 key = make_uint2(static_cast<uint32_t>(pa.seed), static_cast<uint32_t>(pa.seed >> 32));
        const uint32_t c3 = kExploreTag | (static_cast<uint32_t>((EPISODES ? step : t) * P::A + I) *
                                           static_cast<uint32_t>(mlp_explore_stride<P>()));
        uint32_t bits[(AD + 3) / 4 * 4];
#pragma unroll
        for (int b = 0; b < (AD + 3) / 4; ++b) {
            const uint4 r = philox4x32_10(make_uint4(static_cast<uint32_t>(gw), static_cast<uint32_t>(gw >> 32),
                                                     static_cast<uint32_t>(EPISODES ? epoch : pa.epoch),
                                                     c3 | static_cast<uint32_t>(b)), key);
            bits[4 * b] = r.x; bits[4 * b + 1] = r.y; bits[4 * b + 2] = r.z; bits[4 * b + 3] = r.w;
        }
#pragma unroll
        for (int c = 0; c < AD; ++c) {
            const float u = __fmul_rn(__fadd_rz(static_cast<float>(bits[c] >> 8), 0.5f), 0x1p-24f);
            z[c] = __fsub_rn(z[c], logf(-logf(u)));
        }
    }
    float pr[AD];
    if constexpr (CATEGORICAL) {                           // one-hot of the (perturbed) arg-max per sub-space
        constexpr int NSUB = (MOVE > 0) + (COMM > 0);
        int k[NSUB];
        float lp = 0.0f;
        if constexpr (MOVE > 0) lp = categorical_segment<0, MOVE>(z, zl, pr, k[0]);
        if constexpr (COMM > 0) {
            const float lc = categorical_segment<MOVE, COMM>(z, zl, pr, k[NSUB - 1]);
            lp = MOVE > 0 ? __fadd_rn(lp, lc) : lc;
        }
        if (active) {
            if (cr->index[I] != nullptr) {
                int32_t *rec = cr->index[I] + (static_cast<int64_t>(t) * n + wi) * NSUB;
#pragma unroll
                for (int s = 0; s < NSUB; ++s) rec[s] = k[s];
            }
            if (cr->logp != nullptr) cr->logp[(static_cast<int64_t>(t) * P::A + I) * n + wi] = lp;
        }
    } else {
        if constexpr (MOVE > 0) softmax_segment<0, MOVE>(z, pr);
        if constexpr (COMM > 0) softmax_segment<MOVE, COMM>(z, pr);
    }
    if (!CATEGORICAL && pa.act_rec[I] != nullptr && active) {
        float *rec = pa.act_rec[I] + (static_cast<int64_t>(t) * n + wi) * AD;
#pragma unroll
        for (int c = 0; c < AD; ++c) rec[c] = pr[c];
    }
    // _set_action (environment.py:173-190), the arithmetic of decode_rows
    if constexpr (COMM > 0) {
#pragma unroll
        for (int q = 0; q < COMM; ++q) cact[I * P::DIMC + q] = pr[MOVE + q];
    }
    if constexpr (MOVE > 0) {
        return movement_force(pr[1], pr[2], pr[3], pr[4], d.a_sens[I]);
    } else {
        return make_float2(0.0f, 0.0f);                    // immovable: no force, and physics<P> never moves it
    }
}

// register-only observation writers: the sum of an observation's entries, and the sum of their squared deviations from
// mu (P::observe is pure in the world registers, so the critic calls it once per pass)
struct SumWriter {
    float s = 0.0f;
    __device__ __forceinline__ void put(float x) { s += x; }
    __device__ __forceinline__ void put2(float a, float b) { s += a; s += b; }
    __device__ __forceinline__ void put2(float2 v) { put2(v.x, v.y); }
};
struct SqDevWriter {
    float mu, s = 0.0f;
    __device__ __forceinline__ void put(float x) { const float dx = x - mu; s += dx * dx; }
    __device__ __forceinline__ void put2(float a, float b) { put(a); put(b); }
    __device__ __forceinline__ void put2(float2 v) { put2(v.x, v.y); }
};

// Critic W1's columns of agent I ([64][D] torch layout, global) -> TF32 B fragments of its kt1(I) k-tiles, as
// stage_fragments (PERM = false) lays them out; columns beyond obs_dim_I are zero.  K = I: a local critic's W1
// ([64][obs_dim_I]).
template <class P, int I, int K = -1>
__device__ __forceinline__ void stage_critic_w1(float *dst, const float *__restrict__ W) {
    using C = CriticShape<P, K>;
    constexpr int KT = MlpShape<P, 64>::kt1(I), OD = P::obs_dim(I), D = C::in_dim(), OFF = C::col_off(I);
    for (int q = threadIdx.x; q < KT * C::NT * 64; q += blockDim.x) {
        const int j = q & 1, l = (q >> 1) & 31, tile = q >> 6;
        const int nt = tile % C::NT, kt = tile / C::NT;
        const int nn = nt * 8 + (l >> 2);
        const int k = kt * 8 + (l & 3) + 4 * j;
        dst[q] = __uint_as_float(to_tf32(k < OD ? W[nn * D + OFF + k] : 0.0f));
    }
}

// MAPPO's centralized critic for the warp's 32 worlds (MlpCriticState), one weight set Wc (CriticShape): its value of
// row r goes to dst[s * n + r], s < slots, for r < rows.  The input LayerNorm's statistics over all D entries are two
// fp32 passes of register-only writers over every agent's observation; layer 1 then sums, agent by agent, that agent's
// observation in the warp's observation tile, normalised in place, times its k-tiles of W1.  Layers 2 and 3 run as
// MAPPO's actor runs them, one m-tile at a time, with act_norm_tf32_frags; layer 3 has one real output column.  Called
// by all 32 lanes; the tile is free on entry and on return.  K >= 0: IPPO's local critic of agent K (CriticShape<P,
// K>), the same arithmetic on obs_K alone.
template <class P, int K = -1>
__device__ __forceinline__ void mlp_critic(const float *__restrict__ Wc, const DevDesc &d, const typename P::W &w,
                                           float *tile, int lane, int rows, float ln_eps, uint32_t net_flags, float *dst,
                                           int slots, int64_t n) {
    using C = CriticShape<P, K>;
    constexpr int NT = C::NT, D = C::in_dim();
    const int gq = lane >> 2, tq = lane & 3;
    const bool feature_norm = net_flags & kMappoFeatureNorm;
    float mu = 0.0f, rstd = 1.0f;
    if (feature_norm) {
        SumWriter sw;
        static_for<P::A>([&](auto ic) {
            if constexpr (K < 0 || decltype(ic)::value == K) P::template observe<decltype(ic)::value>(d, w, sw);
        });
        mu = sw.s / static_cast<float>(D);
        SqDevWriter vw{mu};
        static_for<P::A>([&](auto ic) {
            if constexpr (K < 0 || decltype(ic)::value == K) P::template observe<decltype(ic)::value>(d, w, vw);
        });
        rstd = rsqrtf(vw.s / static_cast<float>(D) + ln_eps);
    }
    // ---- layer 1: sum over agents of [32 x K1_i] . W1[:, agent i's columns]^T, + b1 ----
    float h[2][NT][4];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
        const float2 b = *reinterpret_cast<const float2 *>(Wc + C::b1_off + nt * 8 + 2 * tq);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) { h[mt][nt][0] = b.x; h[mt][nt][1] = b.y; h[mt][nt][2] = b.x; h[mt][nt][3] = b.y; }
    }
    static_for<P::A>([&](auto ic) {
        constexpr int I = decltype(ic)::value;
        constexpr int OD = P::obs_dim(I), KT1 = MlpShape<P, 64>::kt1(I), PITCH = ObsTile<OD>::kPitch;
        if constexpr (K < 0 || I == K) {
        {
            TileWriter<OD> o(tile, lane);
            P::template observe<I>(d, w, o);
        }
        __syncwarp();
        if (feature_norm) {
            float *row = tile + lane * PITCH;
#pragma unroll
            for (int c = 0; c < OD; ++c) row[c] = (row[c] - mu) * rstd;
            __syncwarp();
        }
        const float *W1 = Wc + C::w1_off(I);
#pragma unroll
        for (int kt = 0; kt < KT1; ++kt) {
            uint32_t a[2][4];
            const int c0 = kt * 8 + tq, c1 = c0 + 4;
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
                const float *r0 = tile + (mt * 16 + gq) * PITCH, *r1 = r0 + 8 * PITCH;
                a[mt][0] = to_tf32(c0 < OD ? r0[c0] : 0.0f); a[mt][1] = to_tf32(c0 < OD ? r1[c0] : 0.0f);
                a[mt][2] = to_tf32(c1 < OD ? r0[c1] : 0.0f); a[mt][3] = to_tf32(c1 < OD ? r1[c1] : 0.0f);
            }
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) {
                const float2 b = *reinterpret_cast<const float2 *>(W1 + ((kt * NT + nt) * 32 + lane) * 2);
                mma_tf32(h[0][nt], a[0], b);
                mma_tf32(h[1][nt], a[1], b);
            }
        }
        __syncwarp();   // every lane has read the tile before the next observation overwrites it
        }
    });
    uint32_t x1[2][NT][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) act_norm_tf32_frags<NT>(x1[mt], h[mt], net_flags & kMappoTanh, ln_eps);
    // ---- layers 2 and 3 per m-tile: h2 = x1 . W2^T + b2, act + LayerNorm, v = x2 . W3^T + b3 ----
    const float *W2 = Wc + C::w2_off, *W3 = Wc + C::w3_off;
    const float2 b3 = *reinterpret_cast<const float2 *>(Wc + C::b3_off + 2 * tq);
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
        float c[NT][4];
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            const float2 bb = *reinterpret_cast<const float2 *>(Wc + C::b2_off + nt * 8 + 2 * tq);
            c[nt][0] = bb.x; c[nt][1] = bb.y; c[nt][2] = bb.x; c[nt][3] = bb.y;
#pragma unroll
            for (int kt = 0; kt < NT; ++kt)
                mma_tf32(c[nt], x1[mt][kt], *reinterpret_cast<const float2 *>(W2 + ((kt * NT + nt) * 32 + lane) * 2));
        }
        uint32_t x2[NT][4];
        act_norm_tf32_frags<NT>(x2, c, net_flags & kMappoTanh, ln_eps);
        float v[4] = {b3.x, b3.y, b3.x, b3.y};
#pragma unroll
        for (int kt = 0; kt < NT; ++kt) mma_tf32(v, x2[kt], *reinterpret_cast<const float2 *>(W3 + (kt * 32 + lane) * 2));
        // column 0 of rows g and g + 8 sits in element 0 and 2 of the quad's first lane
        const int ra = mt * 16 + gq, rb = ra + 8;
        if (tq == 0) {
            for (int s = 0; s < slots; ++s) {
                if (ra < rows) dst[s * n + ra] = v[0];
                if (rb < rows) dst[s * n + rb] = v[2];
            }
        }
        __syncwarp();   // as in MAPPO's actor: the second m-tile reads W2's and W3's fragments again
    }
}

// every critic's values of the current state into record row `row` of rec (values [T][A][n] or final_values):
// a shared critic's (count 1) for every agent, else critic k's for agent k.  LOCAL: agent k's value is V_k(obs_k), from
// the shared critic (count 1) or critic k (LocalCriticShape).
template <class P, bool LOCAL = false>
__device__ __forceinline__ void run_critics(const MlpCriticState &cs, const float *Wc, const DevDesc &d,
                                            const typename P::W &w, float *tile, int lane, int rows, float ln_eps,
                                            uint32_t net_flags, float *rec, int row, int64_t w0, int64_t n) {
    if constexpr (LOCAL) {
        // one agent per iteration: unrolled, the A independent evaluations overlap and spill (spread N=6 at 255
        // registers)
#pragma unroll 1
        for (int k = 0; k < P::A; ++k)
            static_for<P::A>([&](auto kc) {
                constexpr int K = decltype(kc)::value;
                if (K == k)
                    mlp_critic<P, K>(Wc + (cs.count == 1 ? 0 : LocalCriticShape<P>::critic_off(K)), d, w, tile, lane,
                                     rows, ln_eps, net_flags, rec + (static_cast<int64_t>(row) * P::A + K) * n + w0, 1, n);
            });
    } else {
    const int slots = cs.count == 1 ? P::A : 1;
#pragma unroll 1
    for (int k = 0; k < cs.count; ++k)
        mlp_critic<P>(Wc + k * CriticShape<P>::kFloats, d, w, tile, lane, rows, ln_eps, net_flags,
                      rec + (static_cast<int64_t>(row) * P::A + k) * n + w0, slots, n);
    }
}

// Agent I's turn in the separated recurrent actor (SEPARATED): the whole block waits until every warp is done with the
// previous agent's weights, then one thread copies agent I's fragment image into the slot with one TMA bulk copy that
// completes on the mbarrier, and every thread waits for that phase.  phase counts the block's turns mod 2.
template <class P, int I>
__device__ __forceinline__ void gru_restage(float *slot, const float *images, uint64_t *bar, uint32_t &phase) {
    constexpr uint32_t kBytes = GruSeparatedShape<P>::image_floats(I) * 4;
    __syncthreads();
    if (threadIdx.x == 0) {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the slot's generic reads before the async write
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(kBytes) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(smem_u32(slot)), "l"(images + GruSeparatedShape<P>::image_off(I)), "r"(kBytes),
                     "r"(smem_u32(bar)) : "memory");
    }
    uint32_t done;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(smem_u32(bar)), "r"(phase) : "memory");
    } while (!done);
    phase ^= 1u;
}

// the body of both forms; ea is null in the single-episode form (EPISODES = false), cr unless CATEGORICAL; ln_eps and
// net_flags are MAPPO's (MlpMappoArgs), gs the recurrent actor's (GRU, MlpGruArgs), cs the critic's (CRITIC,
// MlpCriticArgs).  SEPARATED (with GRU) gives every agent its own weight set, restaged into one slot from the fragment
// images at `images` (GruSeparatedShape) at every agent's turn (gru_restage).  LOCAL (with CRITIC) makes cs IPPO's local
// critics (LocalCriticShape).
template <class P, int H, bool EPISODES, bool CATEGORICAL = false, bool MAPPO = false, bool GRU = false,
          bool CRITIC = false, bool SEPARATED = false, bool LOCAL = false>
__device__ __forceinline__ void mlp_rollout(const MlpPolicyArgs &pa, const MlpEpisodeArgs *ea,
                                            const MlpCategoricalRecords *cr = nullptr, float ln_eps = 0.0f,
                                            uint32_t net_flags = 0, const MlpGruState *gs = nullptr,
                                            const MlpCriticState *cs = nullptr, const float *images = nullptr) {
    static_assert(!CRITIC || (MAPPO && !GRU), "the critic runs next to MAPPO's MLP actor");
    static_assert(!SEPARATED || GRU, "per-agent weight sets are the recurrent actor's");
    static_assert(!LOCAL || CRITIC, "the local critics are a critic form");
    static_assert(H == 32 || H == 64, "MLP policy rollout: hidden width 32 or 64");
    constexpr int A = P::A, L = P::L, NC = Shape<P>::kNC;
    using S = MlpShape<P, H>;
    constexpr int kWarps = [] {
        if constexpr (SEPARATED) return gru_separated_block_warps<P>();
        else if constexpr (GRU) return gru_block_warps<P>();
        else if constexpr (CRITIC && LOCAL) return local_critic_block_warps<P, EPISODES>();
        else if constexpr (CRITIC) return critic_block_warps<P, EPISODES>();
        else return mlp_block_warps<P, H, EPISODES | (MAPPO ? 2 : CATEGORICAL) << 1>();
    }();
    constexpr int kSlotOff = SEPARATED ? 4 : 0;   // SEPARATED: the slot's mbarrier, then the slot (16-byte aligned)
    constexpr int kWeightFloats = [] {
        if constexpr (SEPARATED) return kSlotOff + GruSeparatedShape<P>::kSlotFloats;
        else if constexpr (GRU) return GruShape<P>::kWeightFloats;
        else return S::kWeightFloats;
    }();
    static_assert(kWarps >= 1 && (kWeightFloats + (CRITIC ? (LOCAL ? LocalCriticShape<P>::kMinFloats : CriticShape<P>::kFloats) : 0) +
                                  kWarps * S::kWarpFloats) * 4 <= kMlpSmemBytes, "one block fits an SM");
    const StepArgs &a = pa.s;
    extern __shared__ __align__(16) float smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint64_t *const bar = reinterpret_cast<uint64_t *>(smem);   // SEPARATED: the slot's mbarrier
    uint32_t phase = 0;                                          // SEPARATED: the block's turns mod 2
    if constexpr (SEPARATED) {    // ---- no weights yet: agent 0's first turn stages them ----
        if (threadIdx.x == 0) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(bar)) : "memory");
    } else if constexpr (GRU) {   // ---- the one shared weight set -> TF32 B fragments in shared memory, once per block ----
        using G = GruShape<P>;
        constexpr int OD = P::obs_dim(0), AD = P::act_dim(0);
        stage_fragments<S::kt1(0), G::NT, false>(smem, pa.w1[0], 64, OD);
        stage_fragments<G::NT, G::NT, true>(smem + G::w2_off, pa.w2[0], 64, 64);
        stage_fragments<G::NT, G::NG, true>(smem + G::wih_off, gs->w_ih, 192, 64);
        stage_fragments<G::NT, G::NG, true>(smem + G::whh_off, gs->w_hh, 192, 64);
        stage_fragments<G::NT, S::nout(0) / 8, true>(smem + G::w3_off, pa.w3[0], AD, 64);
        for (int q = threadIdx.x; q < 64; q += blockDim.x) {
            smem[G::b1_off + q] = pa.b1[0][q];
            smem[G::b2_off + q] = pa.b2[0][q];
        }
        for (int q = threadIdx.x; q < 192; q += blockDim.x) {
            smem[G::bih_off + q] = gs->b_ih[q];
            smem[G::bhh_off + q] = gs->b_hh[q];
        }
        for (int q = threadIdx.x; q < S::nout(0); q += blockDim.x) smem[G::b3_off + q] = q < AD ? pa.b3[0][q] : 0.0f;
    } else {
    // ---- all agents' weights -> TF32 B fragments in shared memory, once per block ----
    static_for<A>([&](auto ic) {
        constexpr int i = decltype(ic)::value;
        constexpr int OD = P::obs_dim(i);
        float *base = smem + S::agent_off(i);
        stage_fragments<S::kt1(i), S::NT, false>(base, pa.w1[i], H, OD);
        stage_fragments<S::NT, S::NT, true>(base + S::w2_off(i), pa.w2[i], H, H);
        stage_fragments<S::NT, S::nout(i) / 8, true>(base + S::w3_off(i), pa.w3[i], P::act_dim(i), H);
        for (int q = threadIdx.x; q < H; q += blockDim.x) {
            base[S::b1_off(i) + q] = pa.b1[i][q];
            base[S::b2_off(i) + q] = pa.b2[i][q];
        }
        for (int q = threadIdx.x; q < S::nout(i); q += blockDim.x) base[S::b3_off(i) + q] = q < P::act_dim(i) ? pa.b3[i][q] : 0.0f;
    });
    }
    int crit_floats = 0;   // the critics' weights after the actor's (CriticShape), cs->count sets
    if constexpr (CRITIC && LOCAL) {   // set k (critic_off(k)) has agent k's W1; the shared set agent 0's
        using LC = LocalCriticShape<P>;
        crit_floats = LC::weight_floats(cs->count);
        static_for<A>([&](auto kc) {
            constexpr int k = decltype(kc)::value;
            using C = CriticShape<P, k>;
            static_assert(C::kFloats == LC::floats(k), "one local critic layout");
            if (k < cs->count) {
                float *base = smem + kWeightFloats + LC::critic_off(k);
                stage_critic_w1<P, k, k>(base, cs->w1[k]);
                stage_fragments<C::NT, C::NT, true>(base + C::w2_off, cs->w2[k], 64, 64);
                stage_fragments<C::NT, 1, true>(base + C::w3_off, cs->w3[k], 1, 64);
                for (int q = threadIdx.x; q < 64; q += blockDim.x) {
                    base[C::b1_off + q] = cs->b1[k][q];
                    base[C::b2_off + q] = cs->b2[k][q];
                }
                for (int q = threadIdx.x; q < 8; q += blockDim.x) base[C::b3_off + q] = q == 0 ? cs->b3[k][0] : 0.0f;
            }
        });
    } else if constexpr (CRITIC) {
        using C = CriticShape<P>;
        crit_floats = cs->count * C::kFloats;
#pragma unroll 1
        for (int k = 0; k < cs->count; ++k) {
            float *base = smem + kWeightFloats + k * C::kFloats;
            static_for<A>([&](auto ic) {
                constexpr int i = decltype(ic)::value;
                stage_critic_w1<P, i>(base + C::w1_off(i), cs->w1[k]);
            });
            stage_fragments<C::NT, C::NT, true>(base + C::w2_off, cs->w2[k], 64, 64);
            stage_fragments<C::NT, 1, true>(base + C::w3_off, cs->w3[k], 1, 64);
            for (int q = threadIdx.x; q < 64; q += blockDim.x) {
                base[C::b1_off + q] = cs->b1[k][q];
                base[C::b2_off + q] = cs->b2[k][q];
            }
            for (int q = threadIdx.x; q < 8; q += blockDim.x) base[C::b3_off + q] = q == 0 ? cs->b3[k][0] : 0.0f;
        }
    }
    __syncthreads();

    const int64_t n = a.n;
    const int64_t end = a.begin + a.count;
    const int64_t w0 = a.begin + (static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + warp) * 32;
    if (w0 >= end) {
        if constexpr (SEPARATED) {   // a warp without worlds still takes part in every turn's barrier
#pragma unroll 1
            for (int e = 0; e < (EPISODES ? ea->episodes : 1); ++e)
#pragma unroll 1
                for (int t = 0; t < pa.T; ++t)
                    static_for<A>([&](auto ic) { gru_restage<P, decltype(ic)::value>(smem + kSlotOff, images, bar, phase); });
        }
        return;
    }
    const int rows = (end - w0) < 32 ? static_cast<int>(end - w0) : 32;
    const bool active = lane < rows;
    const int64_t wi = w0 + (active ? lane : 0);   // idle lanes of a partial tile replay world w0: every tile row is finite
    float *s_warp = smem + kWeightFloats + crit_floats + warp * S::kWarpFloats;
    const float *Wc = smem + kWeightFloats;   // the critics' weights
    const DevDesc &d = a.d;

    typename P::W w;
#pragma unroll
    for (int i = 0; i < A; ++i) {
        const float4 v = a.pv[i * n + wi];
        w.px[i] = v.x; w.py[i] = v.y; w.vx[i] = v.z; w.vy[i] = v.w;
    }
#pragma unroll
    for (int l = 0; l < L; ++l) {
        const float2 v = a.lm[l * n + wi];
        w.lx[l] = v.x; w.ly[l] = v.y;
    }
    if constexpr (P::G > 0) {
#pragma unroll
        for (int q = 0; q < P::G; ++q) w.g[q] = a.goal[q * n + wi];
    }
    if constexpr (NC > 0) {
#pragma unroll
        for (int q = 0; q < NC; ++q) w.c[q] = a.comm[q * n + wi];
    }

    float rsum[A];
#pragma unroll 1
    for (int e = 0; e < (EPISODES ? ea->episodes : 1); ++e) {   // the single-episode form runs one
#pragma unroll
        for (int i = 0; i < A; ++i) rsum[i] = 0.0f;
#pragma unroll 1
        for (int t = 0; t < pa.T; ++t) {
            const int tg = EPISODES ? e * pa.T + t : t;         // the records' step
            float ux[A], uy[A];
            float cact[NC > 0 ? NC : 1];
            P::prepare(d, w);
            if constexpr (CRITIC) run_critics<P, LOCAL>(*cs,Wc, d, w, s_warp, lane, rows, ln_eps, net_flags, cs->values, tg, w0, n);   // V of the state the actors act on
            static_for<A>([&](auto ic) {
                constexpr int i = decltype(ic)::value;
                if constexpr (SEPARATED) gru_restage<P, i>(smem + kSlotOff, images, bar, phase);
                const float2 u = mlp_agent<P, H, i, EPISODES, CATEGORICAL, MAPPO, GRU>(
                    pa, w, GRU ? smem + kSlotOff : smem + S::agent_off(i), s_warp, lane, tg, rows, active, w0, wi, cact, t,
                    pa.epoch + e, cr, ln_eps, net_flags, gs);
                ux[i] = u.x;
                uy[i] = u.y;
            });
            physics<P>(d, w, ux, uy);
#pragma unroll
            for (int q = 0; q < NC; ++q) w.c[q] = cact[q];      // update_agent_state (core.py:171-177), as the fused step
            float rew[A];
            P::reward(d, w, rew, nullptr);
            if (a.flags & MPE_FLAG_SHARED_REWARD) {
                float sum = 0.0f;
#pragma unroll
                for (int i = 0; i < A; ++i) sum += rew[i];
#pragma unroll
                for (int i = 0; i < A; ++i) rew[i] = sum;
            }
#pragma unroll
            for (int i = 0; i < A; ++i) rsum[i] = __fadd_rn(rsum[i], rew[i]);
            if (pa.rew_steps != nullptr && active) {
#pragma unroll
                for (int i = 0; i < A; ++i) pa.rew_steps[(static_cast<int64_t>(tg) * A + i) * n + wi] = rew[i];
            }
        }
        if constexpr (EPISODES) {                          // episode end: returns, final observations, reset
            if (active) {
#pragma unroll
                for (int i = 0; i < A; ++i) a.rew[(static_cast<int64_t>(e) * A + i) * n + wi] = rsum[i];
            }
            if constexpr (CRITIC) {                            // V of the final state, before the reset
                P::prepare(d, w);
                __syncwarp();                                  // every lane has read its logits before the tile is reused
                run_critics<P, LOCAL>(*cs,Wc, d, w, s_warp, lane, rows, ln_eps, net_flags, cs->final_values, e, w0, n);
            }
            if (ea->final_obs[0] != nullptr) {                 // all agents or none (checked by the launcher)
                P::prepare(d, w);
                __syncwarp();                                  // every lane has read its logits before the tile is reused
                static_for<A>([&](auto ic) {
                    constexpr int i = decltype(ic)::value;
                    constexpr int OD = P::obs_dim(i);
                    {
                        TileWriter<OD> o(s_warp, lane);
                        P::template observe<i>(d, w, o);
                    }
                    __syncwarp();
                    store_obs_rows<OD>(ea->final_obs[i] + (static_cast<int64_t>(e) * n + w0) * OD, s_warp, lane, rows, active);
                    __syncwarp();
                });
            }
            struct ToRegs {
                typename P::W &w;
                __device__ void agent(int i, float x, float y) const { w.px[i] = x; w.py[i] = y; w.vx[i] = 0.0f; w.vy[i] = 0.0f; }
                __device__ void landmark(int l, float x, float y) const { w.lx[l] = x; w.ly[l] = y; }
                __device__ void comm(int q) const { w.c[q] = 0.0f; }
                __device__ void goal(int g, int32_t v) const { w.g[g] = v; }
            } out{w};
            draw_initial_state(A, L, NC, P::G, ea->reset_seed, pa.world_offset + static_cast<uint64_t>(wi), ea->reset_epoch + e,
                               reset_landmark_range(P::kScenario), L > 0 ? L : 1, out);
        }
    }
    if (active) {
#pragma unroll
        for (int i = 0; i < A; ++i)                        // the reset moves immovable agents too
            if (EPISODES || P::movable(i)) a.pv[i * n + wi] = make_float4(w.px[i], w.py[i], w.vx[i], w.vy[i]);
        if constexpr (EPISODES) {
#pragma unroll
            for (int l = 0; l < L; ++l) ea->lm[l * n + wi] = make_float2(w.lx[l], w.ly[l]);
#pragma unroll
            for (int q = 0; q < P::G; ++q) ea->goal[q * n + wi] = w.g[q];
        }
#pragma unroll
        for (int q = 0; q < NC; ++q) a.comm[q * n + wi] = w.c[q];
    }
    P::prepare(d, w);
    __syncwarp();                  // every lane has read its logits before the tile is reused
    if constexpr (CRITIC && !EPISODES)
        run_critics<P, LOCAL>(*cs,Wc, d, w, s_warp, lane, rows, ln_eps, net_flags, cs->final_values, 0, w0, n);   // V after the last step
    write_observations<P>(a, d, w, s_warp, lane, rows, active, w0, wi);   // the slot is this warp's observation tile
    if (active) {
#pragma unroll
        for (int i = 0; i < A; ++i) {
            if constexpr (!EPISODES) a.rew[i * n + wi] = rsum[i];
            a.done[i * n + wi] = 0;
        }
    }
}

template <class P, int H>
__global__ void __launch_bounds__(mlp_block_warps<P, H, 0>() * 32) mpe_policy_mlp_rollout_kernel(const __grid_constant__ MlpPolicyArgs pa) {
    mlp_rollout<P, H, false>(pa, nullptr);
}

template <class P, int H>
__global__ void __launch_bounds__(mlp_block_warps<P, H, 1>() * 32)
    mpe_policy_mlp_episode_kernel(const __grid_constant__ MlpEpisodeArgs ea) {
    mlp_rollout<P, H, true>(ea.p, &ea);
}

template <class P, int H>
__global__ void __launch_bounds__(mlp_block_warps<P, H, 2>() * 32)
    mpe_policy_mlp_categorical_kernel(const __grid_constant__ MlpCategoricalArgs ca) {
    mlp_rollout<P, H, false, true>(ca.p, nullptr, &ca.c);
}

template <class P, int H>
__global__ void __launch_bounds__(mlp_block_warps<P, H, 3>() * 32)
    mpe_policy_mlp_categorical_episode_kernel(const __grid_constant__ MlpCategoricalEpisodeArgs ca) {
    mlp_rollout<P, H, true, true>(ca.e.p, &ca.e, &ca.c);
}

template <class P>
__global__ void __launch_bounds__(mlp_block_warps<P, 64, 4>() * 32)
    mpe_policy_mappo_kernel(const __grid_constant__ MlpMappoArgs ma) {
    mlp_rollout<P, 64, false, true, true>(ma.c.p, nullptr, &ma.c.c, ma.eps, ma.net_flags);
}

template <class P>
__global__ void __launch_bounds__(mlp_block_warps<P, 64, 5>() * 32)
    mpe_policy_mappo_episode_kernel(const __grid_constant__ MlpMappoEpisodeArgs ma) {
    mlp_rollout<P, 64, true, true, true>(ma.c.e.p, &ma.c.e, &ma.c.c, ma.eps, ma.net_flags);
}

// MAPPO's actor with its centralized critic (MlpCriticArgs); mpe_critic.cu instantiates them (critic_kernel)
template <class P>
__global__ void __launch_bounds__(critic_block_warps<P, false>() * 32)
    mpe_policy_mappo_critic_kernel(const __grid_constant__ MlpCriticArgs ca) {
    mlp_rollout<P, 64, false, true, true, false, true>(ca.m.c.p, nullptr, &ca.m.c.c, ca.m.eps, ca.m.net_flags, nullptr, &ca.v);
}

template <class P>
__global__ void __launch_bounds__(critic_block_warps<P, true>() * 32)
    mpe_policy_mappo_critic_episode_kernel(const __grid_constant__ MlpCriticEpisodeArgs ca) {
    mlp_rollout<P, 64, true, true, true, false, true>(ca.m.c.e.p, &ca.m.c.e, &ca.m.c.c, ca.m.eps, ca.m.net_flags, nullptr,
                                                      &ca.v);
}

template <class P>
__global__ void __launch_bounds__(gru_block_warps<P>() * 32) mpe_policy_gru_kernel(const __grid_constant__ MlpGruArgs ga) {
    mlp_rollout<P, 64, false, true, true, true>(ga.m.c.p, nullptr, &ga.m.c.c, ga.m.eps, ga.m.net_flags, &ga.g);
}

template <class P>
__global__ void __launch_bounds__(gru_block_warps<P>() * 32)
    mpe_policy_gru_episode_kernel(const __grid_constant__ MlpGruEpisodeArgs ga) {
    mlp_rollout<P, 64, true, true, true, true>(ga.m.c.e.p, &ga.m.c.e, &ga.m.c.c, ga.m.eps, ga.m.net_flags, &ga.g);
}

// Per-agent recurrent actors: agent i's weight set (GruAgentShape<P, i>) -> TF32 B fragments, the layout the shared
// actor stages in shared memory, written to its image in global memory.  Block i writes agent i's image.
template <class P, int I>
__device__ __forceinline__ void stage_gru_agent(float *dst, const float *const (&w)[10]) {
    using G = GruAgentShape<P, I>;
    using S = MlpShape<P, 64>;
    constexpr int OD = P::obs_dim(I), AD = P::act_dim(I);
    stage_fragments<S::kt1(I), G::NT, false>(dst, w[0], 64, OD);
    stage_fragments<G::NT, G::NT, true>(dst + G::w2_off, w[2], 64, 64);
    stage_fragments<G::NT, G::NG, true>(dst + G::wih_off, w[4], 192, 64);
    stage_fragments<G::NT, G::NG, true>(dst + G::whh_off, w[6], 192, 64);
    stage_fragments<G::NT, S::nout(I) / 8, true>(dst + G::w3_off, w[8], AD, 64);
    for (int q = threadIdx.x; q < 64; q += blockDim.x) {
        dst[G::b1_off + q] = w[1][q];
        dst[G::b2_off + q] = w[3][q];
    }
    for (int q = threadIdx.x; q < 192; q += blockDim.x) {
        dst[G::bih_off + q] = w[5][q];
        dst[G::bhh_off + q] = w[7][q];
    }
    for (int q = threadIdx.x; q < G::kImageFloats - G::b3_off; q += blockDim.x) dst[G::b3_off + q] = q < AD ? w[9][q] : 0.0f;
}
constexpr int kGruImageThreads = 256;
template <class P>
__global__ void __launch_bounds__(kGruImageThreads) mpe_gru_image_kernel(const __grid_constant__ GruImageArgs ia) {
    static_for<P::A>([&](auto ic) {
        constexpr int i = decltype(ic)::value;
        static_assert(GruSeparatedShape<P>::image_floats(i) == GruAgentShape<P, i>::kImageFloats, "one image layout");
        if (blockIdx.x == i) {
            const float *const w[10] = {ia.w[0][i], ia.w[1][i], ia.w[2][i], ia.w[3][i], ia.w[4][i],
                                        ia.w[5][i], ia.w[6][i], ia.w[7][i], ia.w[8][i], ia.w[9][i]};
            stage_gru_agent<P, i>(ia.images + GruSeparatedShape<P>::image_off(i), w);
        }
    });
}

template <class P>
__global__ void __launch_bounds__(gru_separated_block_warps<P>() * 32)
    mpe_policy_gru_separated_kernel(const __grid_constant__ MlpGruSeparatedArgs sa) {
    mlp_rollout<P, 64, false, true, true, true, false, true>(sa.g.m.c.p, nullptr, &sa.g.m.c.c, sa.g.m.eps, sa.g.m.net_flags,
                                                             &sa.g.g, nullptr, sa.images);
}

template <class P>
__global__ void __launch_bounds__(gru_separated_block_warps<P>() * 32)
    mpe_policy_gru_separated_episode_kernel(const __grid_constant__ MlpGruSeparatedEpisodeArgs sa) {
    mlp_rollout<P, 64, true, true, true, true, false, true>(sa.g.m.c.e.p, &sa.g.m.c.e, &sa.g.m.c.c, sa.g.m.eps,
                                                            sa.g.m.net_flags, &sa.g.g, nullptr, sa.images);
}

// The recurrent actor's two kernels of program P (episodes = 0, 1).  mpe_gru.cu defines it and so instantiates the 14
// kernels in a translation unit of their own, which the Makefile compiles alongside this one: in one unit the library
// took half as long again to build.
template <class P>
const void *gru_kernel(int episodes);
// The critic's two kernels of program P (episodes = 0, 1), instantiated by mpe_critic.cu in the same way
template <class P>
const void *critic_kernel(int episodes);
// rMAPPO's recurrent critic of program P (RCriticArgs), one kernel for both forms; mpe_critic_gru.cu defines and
// instantiates it for the programs of GruBuilt
template <class P>
const void *critic_gru_kernel();
// IPPO's local critics: MAPPO's actor with them (MlpCriticArgs, episodes = 0, 1) for the programs of
// local_critic_built, and the recurrent local critic (RCriticArgs) for those of GruBuilt.  mpe_critic_local.cu
// defines and instantiates both.
template <class P>
const void *local_critic_kernel(int episodes);
template <class P>
const void *critic_gru_local_kernel();
// The per-agent recurrent actors' kernels of program P: 0 the fragment images, 1 the rollout, 2 its episode form, 3
// rMAPPO's per-agent recurrent critics (RCriticSeparatedArgs).  mpe_gru_separated.cu defines and instantiates it for the
// programs of GruSeparatedBuilt.
template <class P>
const void *gru_separated_kernel(int which);

// MAPPO's GAE over a finished buffer (mpe_gae): one thread per (agent, world) column of [T][A][N], walking t backwards.
// mpe_gae.cu defines the kernels; gae_kernel(0) is the scan, gae_kernel(1) the scan that also sums the advantages and
// their squares (fp64) into the workspace and, in its last block, writes (mean, std), gae_kernel(2) the in-place
// normalisation of the advantages.
constexpr uint32_t kGaeBootstrap = MPE_GAE_BOOTSTRAP, kGaeNormalize = MPE_GAE_NORMALIZE,
                   kGaePerAgentNorm = MPE_GAE_PER_AGENT_VALUE_NORM;
constexpr int kGaeThreads = 128;       // scan block: one fp64 partial (two doubles of workspace) per block
constexpr int kGaeNormThreads = 256;   // normalisation block
constexpr int64_t kGaeWsHeader = 32;   // workspace: double (mean, std) at 0, the uint32 ticket at 16, partials at 32
struct GaeArgs {
    const float *rew, *val;      // [T][A][N]
    const float *final_val;      // [E][A][N], null without kGaeBootstrap
    const float *value_norm;     // (mean, std): [2], [A][2] with kGaePerAgentNorm, or null
    float *ret, *adv;            // [T][A][N]
    double *stats;               // workspace: (mean, std) of the raw advantages
    unsigned *ticket;            // workspace: blocks done with their partial (zeroed before the scan)
    double *partial;             // workspace: [gridDim.x][2] (sum a, sum a^2) per scan block, as two doubles: the
                                 // workspace need only be 8-byte aligned
    int64_t cols, n;             // A * N, N
    int32_t T, L;                // steps, episode length (T for one episode)
    float gamma, lambda;
    uint32_t flags;
};
const void *gae_kernel(int which);

#ifdef MPE_KERNEL_TEMPLATES_ONLY   // mpe_gru.cu: the device code above, without the programs and the C ABI below
}  // namespace mpe
#else
// ---- generic program for user scenarios (MPE_SCN_CUSTOM) ------------------------------------------
// Any entity table, flags read at run time; same arithmetic primitives and the same (a, b) pair order as
// the compiled programs, so for a table that matches a built-in scenario the state is bit-identical.
// Loops are unrolled to the maximum counts with run-time guards, which keeps every array in registers.
__global__ void __launch_bounds__(128) generic_set_action_kernel(const __grid_constant__ StepArgs a) {
    const int64_t w = a.begin + static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (w >= a.begin + a.count) return;
    const DevDesc &d = a.d;
    const int64_t n = a.n;
    const int C = d.g_dim_c;
#pragma unroll
    for (int i = 0; i < kMaxA; ++i) {
        if (i >= d.g_agents) break;
        const bool movable = (d.g_movable >> i) & 1u, silent = (d.g_silent >> i) & 1u;
        const int adim = (movable ? 5 : 0) + (silent ? 0 : C);
        float x = 0.0f, y = 0.0f;
        int off = 0;
        if (a.flags & MPE_FLAG_DISCRETE_ACTION_INPUT) {            // environment.py:161-167, 185-187
            const int nsub = (movable ? 1 : 0) + (silent ? 0 : 1);
            const int32_t *irow = reinterpret_cast<const int32_t *>(a.act[i]) + w * nsub;
            if (movable) {
                const int k = irow[0];
                x = __fmul_rn(k == 1 ? -1.0f : (k == 2 ? 1.0f : 0.0f), d.a_sens[i]);
                y = __fmul_rn(k == 3 ? -1.0f : (k == 4 ? 1.0f : 0.0f), d.a_sens[i]);
                off = 1;
            }
            a.u[i * n + w] = make_float2(x, y);
            if (!silent) {
                const int k = irow[off];
                for (int q = 0; q < C; ++q) a.c[(d.g_slot[i] * C + q) * n + w] = (k == q) ? 1.0f : 0.0f;
            }
            continue;
        }
        const float *row = a.act[i] + w * adim;
        if (movable) {                                             // environment.py:157-181
            float p0 = row[0], p1 = row[1], p2 = row[2], p3 = row[3], p4 = row[4];
            if (a.flags & MPE_FLAG_FORCE_DISCRETE_ACTION) {
                int best = 0;
                float bv = p0;
                if (p1 > bv) { bv = p1; best = 1; }
                if (p2 > bv) { bv = p2; best = 2; }
                if (p3 > bv) { bv = p3; best = 3; }
                if (p4 > bv) { bv = p4; best = 4; }
                p1 = best == 1 ? 1.0f : 0.0f; p2 = best == 2 ? 1.0f : 0.0f;
                p3 = best == 3 ? 1.0f : 0.0f; p4 = best == 4 ? 1.0f : 0.0f;
            }
            x = __fmul_rn(p1 - p2, d.a_sens[i]);
            y = __fmul_rn(p3 - p4, d.a_sens[i]);
            off = 5;
        }
        a.u[i * n + w] = make_float2(x, y);
        if (!silent)                                               // environment.py:183-190
            for (int q = 0; q < C; ++q) a.c[(d.g_slot[i] * C + q) * n + w] = row[off + q];
    }
}

__global__ void __launch_bounds__(128) generic_world_step_kernel(const __grid_constant__ StepArgs a) {
    const int64_t w = a.begin + static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (w >= a.begin + a.count) return;
    const DevDesc &d = a.d;
    const int64_t n = a.n;
    const int A = d.g_agents, L = d.g_landmarks, C = d.g_dim_c;
    float px[kMaxA], py[kMaxA], vx[kMaxA], vy[kMaxA], fx[kMaxA], fy[kMaxA], lx[kMaxL], ly[kMaxL];
#pragma unroll
    for (int i = 0; i < kMaxA; ++i) {
        px[i] = py[i] = vx[i] = vy[i] = fx[i] = fy[i] = 0.0f;
        if (i < A) {
            const float4 v = a.pv[i * n + w];
            const float2 u = a.u[i * n + w];
            px[i] = v.x; py[i] = v.y; vx[i] = v.z; vy[i] = v.w;
            fx[i] = u.x; fy[i] = u.y;                               // apply_action_force (core.py:134-140)
        }
    }
#pragma unroll
    for (int l = 0; l < kMaxL; ++l) {
        lx[l] = ly[l] = 0.0f;
        if (l < L) {
            const float2 v = a.lm[l * n + w];
            lx[l] = v.x; ly[l] = v.y;
        }
    }
    // apply_environment_force (core.py:143-155), pairs (a, b), a < b, agents then landmarks
#pragma unroll
    for (int i = 0; i < kMaxA; ++i) {
        if (i >= A || !((d.g_collide >> i) & 1u)) continue;
#pragma unroll
        for (int j = i + 1; j < kMaxA; ++j) {
            if (j >= A || !((d.g_collide >> j) & 1u)) continue;
            const float2 f = pair_force(__fsub_rn(px[i], px[j]), __fsub_rn(py[i], py[j]), __fadd_rn(d.a_size[i], d.a_size[j]),
                                        d.contact_force, d.contact_margin, d.inv_margin);
            if ((d.g_movable >> i) & 1u) { fx[i] = __fadd_rn(fx[i], f.x); fy[i] = __fadd_rn(fy[i], f.y); }
            if ((d.g_movable >> j) & 1u) { fx[j] = __fsub_rn(fx[j], f.x); fy[j] = __fsub_rn(fy[j], f.y); }
        }
#pragma unroll
        for (int l = 0; l < kMaxL; ++l) {
            if (l >= L || !((d.g_lcollide >> l) & 1u)) continue;
            const float2 f = pair_force(__fsub_rn(px[i], lx[l]), __fsub_rn(py[i], ly[l]), __fadd_rn(d.a_size[i], d.l_size[l]),
                                        d.contact_force, d.contact_margin, d.inv_margin);
            if ((d.g_movable >> i) & 1u) { fx[i] = __fadd_rn(fx[i], f.x); fy[i] = __fadd_rn(fy[i], f.y); }
        }
    }
    // integrate_state (core.py:158-169)
#pragma unroll
    for (int i = 0; i < kMaxA; ++i) {
        if (i >= A || !((d.g_movable >> i) & 1u)) continue;
        float4 r;
        if (d.a_max_speed[i] >= 0.0f)
            r = integrate_entity<true>(px[i], py[i], vx[i], vy[i], fx[i], fy[i], d.keep, d.a_dt_over_mass[i], d.dt, d.a_max_speed[i]);
        else
            r = integrate_entity<false>(px[i], py[i], vx[i], vy[i], fx[i], fy[i], d.keep, d.a_dt_over_mass[i], d.dt, 0.0f);
        a.pv[i * n + w] = r;
    }
    // update_agent_state (core.py:171-177): state.c = action.c for the speakers
    for (int q = 0; q < d.g_comm_rows; ++q) a.comm[q * n + w] = a.c[q * n + w];
    (void)C;
}

// ---- reset: i.i.d. uniform positions (e.g. simple_spread.py:38-45) -----------------------------
struct ResetArgs {
    int64_t n;
    int A, L, NC, G;
    float4 *pv;
    float2 *lm;
    float *comm;
    int32_t *goal;
    const uint8_t *mask;
    uint64_t seed, world_offset, epoch;
    const unsigned long long *epoch_dev;   // when non-null the epoch is read from device memory
    float landmark_range;
    uint32_t goal_mod;
};

__global__ void __launch_bounds__(256) reset_kernel(const __grid_constant__ ResetArgs a) {
    const int64_t w = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (w >= a.n) return;
    if (a.mask != nullptr && a.mask[w] == 0) return;
    struct ToState {
        const ResetArgs &a;
        int64_t w;
        __device__ void agent(int i, float x, float y) const { a.pv[i * a.n + w] = make_float4(x, y, 0.0f, 0.0f); }
        __device__ void landmark(int l, float x, float y) const { a.lm[l * a.n + w] = make_float2(x, y); }
        __device__ void comm(int q) const { a.comm[q * a.n + w] = 0.0f; }
        __device__ void goal(int g, int32_t v) const { a.goal[g * a.n + w] = v; }
    } out{a, w};
    draw_initial_state(a.A, a.L, a.NC, a.G, a.seed, a.world_offset + static_cast<uint64_t>(w),
                       a.epoch_dev ? *a.epoch_dev : a.epoch, a.landmark_range, a.goal_mod, out);
}

__global__ void bump_epoch_kernel(unsigned long long *epoch) { *epoch += 1ull; }

// ---- diagnostics: a pure streaming kernel with a step's byte counts (bench.py's size-matched ceiling) ------
// Reads n_read4 float4, then writes n_write4 float4 that depend on what was read (like a step: stores follow the
// loads), same launch path (programmatic dependent launch) and the same evict-first stores as the step kernel.
__global__ void __launch_bounds__(256) stream_probe_kernel(const float4 *__restrict__ src, long long n_read4,
                                                           float4 *__restrict__ dst, long long n_write4) {
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const long long tid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    const long long nth = static_cast<long long>(gridDim.x) * blockDim.x;
    float acc = 0.0f;
#pragma unroll 8
    for (long long i = tid; i < n_read4; i += nth) {
        const float4 v = src[i];
        acc += (v.x + v.y) + (v.z + v.w);
    }
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const float4 o = make_float4(acc, acc, acc, acc);
#pragma unroll 8
    for (long long i = tid; i < n_write4; i += nth) __stcs(dst + i, o);
}

// ---- program table -----------------------------------------------------------------------------
typedef void (*KernelFn)(StepArgs);

struct Program {
    int scenario;
    bool (*validate)(const mpe_desc &);
    KernelFn fn[4];
    int smem_bytes;  // dynamic shared memory per WARP
    KernelFn hot_fn;    // fused step specialised for whole tiles / float actions / cp.async staging (null: no such program)
    KernelFn hot_dense_fn;   // the same compiled for 80 registers (large batches of programs that fit without spilling)
    void (*policy_fn[2])(PolicyArgs);  // K-step closed-loop rollout, hidden width 32 / 64 (null: not built for this program)
    int policy_weight_floats[2];
    // the same with the two-hidden-layer actor on the tensor cores, by form (episodes | kind << 1) and H = 32 / 64: the
    // kernel and its warps per block at most (mlp_block_warps); null for MAPPO's forms at H = 32.  Forms 6 and 7 are
    // the recurrent actor's (gru_block_warps, H = 64 only), whose one shared weight set takes gru_weight_floats; forms
    // 8 and 9 MAPPO's actor with its critic (critic_block_warps, H = 64 only), each critic taking critic_floats more;
    // 10 and 11 MAPPO's actor with IPPO's local critics (local_critic_block_warps), whose weights take
    // local_critic_floats[0] for one shared critic (0: the agents observe differently, no shared critic) and
    // local_critic_floats[1] for A.
    struct { const void *fn; int warps; } mlp[kMlpForms + 6][2];
    int mlp_weight_floats[2], mlp_warp_floats[2], gru_weight_floats, critic_floats, local_critic_floats[2];
    const void *critic_gru_fn;   // rMAPPO's recurrent critic (kRCriticWarps per block), its weights critic_gru_floats
    int critic_gru_floats;
    const void *critic_gru_local_fn;   // rIPPO's recurrent local critic (kRCriticWarps per block, A blocks in y)
    int critic_gru_local_floats;
    // per-agent recurrent actors and critics (GruSeparatedBuilt, gru_separated_kernel): the fragment images' kernel, the
    // rollout's two forms (kGruWarps per block, a 4-float mbarrier header and gru_sep_slot_floats of slot), the critics
    // (kRCriticWarps per block, critic_gru_floats each); null where not built
    const void *gru_sep_fn[4];
    int gru_sep_slot_floats;
    int64_t gru_sep_image_bytes;   // all agents' fragment images, the workspace the rollout needs
    int mlp_explore_stride;           // Philox blocks per (step, agent) of its exploration noise
    void (*rollout_fn)(RolloutArgs);   // K-step open-loop rollout
    int rollout_smem;   // dynamic shared memory per WARP of the rollout kernel
    int A, L, NS, DIMC, INFO, G;
    int obs_dim[kMaxA], act_dim[kMaxA];
    int unread_state_floats;   // state floats per world that this scenario's step never needs (not compulsory traffic)
};

template <class P, int H>
static void set_mlp(Program &p, int k) {
    p.mlp[0][k] = {reinterpret_cast<const void *>(mpe_policy_mlp_rollout_kernel<P, H>), mlp_block_warps<P, H, 0>()};
    p.mlp[1][k] = {reinterpret_cast<const void *>(mpe_policy_mlp_episode_kernel<P, H>), mlp_block_warps<P, H, 1>()};
    p.mlp[2][k] = {reinterpret_cast<const void *>(mpe_policy_mlp_categorical_kernel<P, H>), mlp_block_warps<P, H, 2>()};
    p.mlp[3][k] = {reinterpret_cast<const void *>(mpe_policy_mlp_categorical_episode_kernel<P, H>), mlp_block_warps<P, H, 3>()};
    if constexpr (H == 64) {
        p.mlp[4][k] = {reinterpret_cast<const void *>(mpe_policy_mappo_kernel<P>), mlp_block_warps<P, H, 4>()};
        p.mlp[5][k] = {reinterpret_cast<const void *>(mpe_policy_mappo_episode_kernel<P>), mlp_block_warps<P, H, 5>()};
    }
    p.mlp_weight_floats[k] = MlpShape<P, H>::kWeightFloats;
    p.mlp_warp_floats[k] = MlpShape<P, H>::kWarpFloats;
}

template <class P>
static Program make_program() {
    Program p{};
    p.scenario = P::kScenario;
    p.validate = &P::validate;
    p.fn[kFusedStep] = mpe_kernel<P, kFusedStep>;
    p.fn[kSetAction] = mpe_kernel<P, kSetAction>;
    p.fn[kWorldStep] = mpe_kernel<P, kWorldStep>;
    p.fn[kObserve] = mpe_kernel<P, kObserve>;
    if constexpr (Shape<P>::all_act_dense()) p.hot_fn = mpe_kernel<P, kFusedStep, true>;
    if constexpr (Shape<P>::all_act_dense() && P::kLowRegVariant) p.hot_dense_fn = mpe_kernel<P, kFusedStep, true, true>;
    p.rollout_fn = mpe_rollout_kernel<P>;
    p.rollout_smem = Shape<P>::kRolloutWarpBytes;
    // the closed-loop rollout is built for the BASELINE.json scenarios whose agents all move and are silent
    if constexpr (policy_rollout_ok<P>() && PolicyBuilt<P>::value) {
        p.policy_fn[0] = mpe_policy_rollout_kernel<P, 32>;
        p.policy_fn[1] = mpe_policy_rollout_kernel<P, 64>;
        p.policy_weight_floats[0] = PolicyShape<P, 32>::kWeightFloats;
        p.policy_weight_floats[1] = PolicyShape<P, 64>::kWeightFloats;
    }
    if constexpr (MlpBuilt<P>::value) {
        set_mlp<P, 32>(p, 0);
        set_mlp<P, 64>(p, 1);
        p.mlp_explore_stride = mlp_explore_stride<P>();
    }
    if constexpr (GruBuilt<P>::value) {
        static_assert(MlpBuilt<P>::value, "the recurrent actor shares the MLP actor's tiles and exploration stride");
        p.mlp[kMlpForms][1] = {gru_kernel<P>(0), gru_block_warps<P>()};
        p.mlp[kMlpForms + 1][1] = {gru_kernel<P>(1), gru_block_warps<P>()};
        p.gru_weight_floats = GruShape<P>::kWeightFloats;
    }
    if constexpr (critic_built<P>()) {
        p.mlp[kMlpForms + 2][1] = {critic_kernel<P>(0), critic_block_warps<P, false>()};
        p.mlp[kMlpForms + 3][1] = {critic_kernel<P>(1), critic_block_warps<P, true>()};
        p.critic_floats = CriticShape<P>::kFloats;
    }
    if constexpr (local_critic_built<P>()) {
        p.mlp[kMlpForms + 4][1] = {local_critic_kernel<P>(0), local_critic_block_warps<P, false>()};
        p.mlp[kMlpForms + 5][1] = {local_critic_kernel<P>(1), local_critic_block_warps<P, true>()};
        p.local_critic_floats[0] = LocalCriticShape<P>::shared_ok() ? LocalCriticShape<P>::weight_floats(1) : 0;
        p.local_critic_floats[1] = LocalCriticShape<P>::weight_floats(P::A);
    }
    if constexpr (GruBuilt<P>::value) {
        p.critic_gru_fn = critic_gru_kernel<P>();
        p.critic_gru_floats = RCriticShape<P>::kFloats;
        p.critic_gru_local_fn = critic_gru_local_kernel<P>();
        p.critic_gru_local_floats = RCriticShape<P, 0>::kFloats;
    }
    if constexpr (GruSeparatedBuilt<P>::value) {
        for (int j = 0; j < 4; ++j) p.gru_sep_fn[j] = gru_separated_kernel<P>(j);
        p.gru_sep_slot_floats = GruSeparatedShape<P>::kSlotFloats;
        p.gru_sep_image_bytes = static_cast<int64_t>(GruSeparatedShape<P>::kImagesFloats) * 4;
        p.critic_gru_floats = RCriticShape<P>::kFloats;
    }
    p.smem_bytes = Shape<P>::kWarpBytes;  // per warp
    p.A = P::A; p.L = P::L; p.NS = P::NS; p.DIMC = P::DIMC; p.INFO = P::INFO; p.G = P::G;
    for (int i = 0; i < P::A; ++i) { p.obs_dim[i] = P::obs_dim(i); p.act_dim[i] = P::act_dim(i); }
    // simple_crypto never looks at a position (nobody moves, observations and rewards are about utterances only);
    // simple_speaker_listener never looks at the immovable speaker's position
    p.unread_state_floats = P::kScenario == MPE_SCN_CRYPTO ? 4 * P::A + 2 * P::L
                          : (P::kScenario == MPE_SCN_SPEAKER_LISTENER ? 4 : 0);
    return p;
}

// MPE_SCN_CUSTOM: shapes come from the descriptor at create time (see mpe_create)
static Program make_generic_program() {
    Program p{};
    p.scenario = MPE_SCN_CUSTOM;
    p.validate = [](const mpe_desc &) { return true; };
    p.fn[kSetAction] = generic_set_action_kernel;
    p.fn[kWorldStep] = generic_world_step_kernel;
    p.smem_bytes = 0;
    return p;
}

static const Program *programs(int *count) {
    static const Program table[] = {
        make_generic_program(),
        make_program<Simple<1, 1>>(),
        make_program<Spread<2>>(), make_program<Spread<3>>(), make_program<Spread<4>>(),
        make_program<Spread<5>>(), make_program<Spread<6>>(),
        make_program<Tag<3, 1, 2>>(), make_program<Tag<1, 1, 2>>(), make_program<Tag<2, 1, 2>>(),
        make_program<Tag<4, 2, 2>>(), make_program<Tag<6, 2, 3>>(),
        make_program<WorldComm<4, 2, 1, 2>>(),
        make_program<Adversary<1, 2, 2>>(), make_program<Adversary<1, 3, 3>>(),
        make_program<Push<1, 1, 2>>(),
        make_program<SpeakerListener>(),
        make_program<Reference>(),
        make_program<Crypto>(),
    };
    *count = static_cast<int>(sizeof(table) / sizeof(table[0]));
    return table;
}

}  // namespace mpe

// =================================================================================================
// C ABI
// =================================================================================================
using namespace mpe;

namespace {
struct NvtxRange {   // RAII range around the C-ABI entry points (visible in nsys / ncu --nvtx)
    explicit NvtxRange(const char *name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
};
}  // namespace

// largest block (in warps) whose warp-private staging fits the 227 KB of dynamic shared memory of an SM
static int max_warps_per_block(int smem_per_warp) {
    const int fit = (227 * 1024) / (smem_per_warp > 0 ? smem_per_warp : 1);
    return fit < 1 ? 1 : (fit > kMaxWarpsPerBlock ? kMaxWarpsPerBlock : fit);
}

static_assert(sizeof(mpe_desc) == 480, "mpe_desc layout is part of the ABI (mirrored by _lib.MpeDesc)");

struct mpe_env {
    mpe_desc desc;
    DevDesc dev;
    Program custom;        // MPE_SCN_CUSTOM: the generic program with this handle's shapes
    const Program *prog;
    int64_t n;
    int device;
    int sms = 0;           // streaming multiprocessors of that device (launch-geometry heuristics)
    // mpe_step_host pipelines chunks of the batch over two internal streams so that the H2D copy of one
    // chunk overlaps the D2H copy of the previous one (PCIe is full duplex)
    cudaStream_t aux[2] = {nullptr, nullptr};
    cudaEvent_t ev_fork = nullptr, ev_join[2] = {nullptr, nullptr};
};

static thread_local char g_cuda_err[256] = "";
static long long g_launches = 0;

static int cuda_fail(cudaError_t e, const char *what) {
    snprintf(g_cuda_err, sizeof(g_cuda_err), "%s: %s", what, cudaGetErrorString(e));
    return MPE_ERR_CUDA;
}
#define CUDA_TRY(expr)                                     \
    do {                                                   \
        cudaError_t e_ = (expr);                           \
        if (e_ != cudaSuccess) return cuda_fail(e_, #expr); \
    } while (0)

extern "C" int mpe_create(const mpe_desc *desc, int64_t n_env, int device, mpe_handle *out) {
    if (!desc || !out || n_env <= 0) return MPE_ERR_BAD_ARG;
    if (desc->abi_version != MPE_ABI_VERSION) return MPE_ERR_BAD_DESC;
    if (desc->n_agents < 1 || desc->n_agents > MPE_MAX_AGENTS || desc->n_landmarks < 0 ||
        desc->n_landmarks > MPE_MAX_LANDMARKS)
        return MPE_ERR_BAD_DESC;
    int count = 0;
    const Program *tab = programs(&count);
    const Program *prog = nullptr;
    bool scenario_known = false;
    for (int i = 0; i < count; ++i) {
        if (tab[i].scenario != desc->scenario) continue;
        scenario_known = true;
        if (tab[i].validate(*desc)) { prog = &tab[i]; break; }
    }
    if (!prog) return scenario_known ? MPE_ERR_BAD_DESC : MPE_ERR_UNSUPPORTED;
    int sms = 0;
    if (device != -1) {  // device == -1: shape-only handle (no CUDA call is made; launches are refused)
        int ndev = 0;
        if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) return MPE_ERR_NO_DEVICE;
        int major = 0, minor = 0;
        CUDA_TRY(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
        CUDA_TRY(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device));
        if (major != 9 || minor != 0) return MPE_ERR_NO_DEVICE;  // sm_90a cubin only
        CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
        int prev = 0;
        CUDA_TRY(cudaGetDevice(&prev));
        CUDA_TRY(cudaSetDevice(device));
        for (int m = 0; m < 4; ++m)
            if (prog->fn[m] && prog->smem_bytes > 0)
                CUDA_TRY(cudaFuncSetAttribute(prog->fn[m], cudaFuncAttributeMaxDynamicSharedMemorySize,
                                              prog->smem_bytes * max_warps_per_block(prog->smem_bytes)));
        if (prog->hot_fn && prog->smem_bytes > 0)
            CUDA_TRY(cudaFuncSetAttribute(prog->hot_fn, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          prog->smem_bytes * max_warps_per_block(prog->smem_bytes)));
        if (prog->hot_dense_fn && prog->smem_bytes > 0)
            CUDA_TRY(cudaFuncSetAttribute(prog->hot_dense_fn, cudaFuncAttributeMaxDynamicSharedMemorySize, prog->smem_bytes * 4));
        for (int k = 0; k < 2; ++k)
            if (prog->policy_fn[k])
                CUDA_TRY(cudaFuncSetAttribute(prog->policy_fn[k], cudaFuncAttributeMaxDynamicSharedMemorySize,
                                              prog->policy_weight_floats[k] * 4 + prog->smem_bytes * 4));
        for (int f = 0; f < kMlpForms + 2; ++f)   // and the recurrent actor's two, whose weights are gru_weight_floats
            for (int k = 0; k < 2; ++k)
                if (prog->mlp[f][k].fn)
                    CUDA_TRY(cudaFuncSetAttribute(prog->mlp[f][k].fn, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                  ((f < kMlpForms ? prog->mlp_weight_floats[k] : prog->gru_weight_floats) +
                                                   prog->mlp_warp_floats[k] * prog->mlp[f][k].warps) * 4));
        for (int f = kMlpForms + 2; f < kMlpForms + 6; ++f)   // the critics' four: their size depends on the critics'
            if (prog->mlp[f][1].fn)                            // count, so they may take the whole opt-in
                CUDA_TRY(cudaFuncSetAttribute(prog->mlp[f][1].fn, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                              kMlpSmemBytes));
        if (prog->critic_gru_fn)
            CUDA_TRY(cudaFuncSetAttribute(prog->critic_gru_fn, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          prog->critic_gru_floats * 4));
        if (prog->critic_gru_local_fn)
            CUDA_TRY(cudaFuncSetAttribute(prog->critic_gru_local_fn, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          prog->critic_gru_local_floats * 4));
        for (int j = 1; j < 3; ++j)
            if (prog->gru_sep_fn[j])
                CUDA_TRY(cudaFuncSetAttribute(prog->gru_sep_fn[j], cudaFuncAttributeMaxDynamicSharedMemorySize,
                                              (4 + prog->gru_sep_slot_floats + kGruWarps * prog->mlp_warp_floats[1]) * 4));
        if (prog->gru_sep_fn[3])
            CUDA_TRY(cudaFuncSetAttribute(prog->gru_sep_fn[3], cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          prog->critic_gru_floats * 4));
        if (prog->rollout_fn)
            CUDA_TRY(cudaFuncSetAttribute(prog->rollout_fn, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          prog->rollout_smem * max_warps_per_block(prog->rollout_smem)));
        CUDA_TRY(cudaSetDevice(prev));
    }

    mpe_env *h = new (std::nothrow) mpe_env();
    if (!h) return MPE_ERR_BAD_ARG;
    if (device != -1) {
        int prev = 0;
        cudaGetDevice(&prev);
        cudaSetDevice(device);
        cudaError_t e = cudaSuccess;
        for (int k = 0; k < 2 && e == cudaSuccess; ++k) {
            e = cudaStreamCreateWithFlags(&h->aux[k], cudaStreamNonBlocking);
            if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->ev_join[k], cudaEventDisableTiming);
        }
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming);
        cudaSetDevice(prev);
        if (e != cudaSuccess) { delete h; return cuda_fail(e, "mpe_create: streams/events"); }
    }
    h->desc = *desc;
    h->prog = prog;
    if (desc->scenario == MPE_SCN_CUSTOM) {   // shapes of a user scenario come from its descriptor
        h->custom = *prog;
        Program &c = h->custom;
        c.A = desc->n_agents; c.L = desc->n_landmarks; c.DIMC = desc->dim_c; c.INFO = 0; c.G = 0; c.NS = 0;
        for (int i = 0; i < c.A; ++i) {
            c.NS += desc->agent_silent[i] ? 0 : 1;
            c.act_dim[i] = (desc->agent_movable[i] ? 5 : 0) + (desc->agent_silent[i] ? 0 : desc->dim_c);
            c.obs_dim[i] = 0;   // defined by the caller's observation code
        }
        h->prog = &h->custom;
    }
    h->n = n_env;
    h->device = device;
    h->sms = sms;
    DevDesc &d = h->dev;
    memset(&d, 0, sizeof(d));
    d.dt = static_cast<float>(desc->dt);
    d.keep = static_cast<float>(1.0 - desc->damping);
    d.contact_force = static_cast<float>(desc->contact_force);
    d.contact_margin = static_cast<float>(desc->contact_margin);
    d.inv_margin = static_cast<float>(1.0 / desc->contact_margin);
    for (int i = 0; i < desc->n_agents; ++i) {
        d.a_size[i] = static_cast<float>(desc->agent_size[i]);
        d.a_dt_over_mass[i] = static_cast<float>(desc->dt / desc->agent_mass[i]);
        d.a_sens[i] = static_cast<float>(desc->agent_sens[i]);
        d.a_max_speed[i] = desc->agent_max_speed[i] < 0 ? -1.0f : static_cast<float>(desc->agent_max_speed[i]);
    }
    for (int l = 0; l < desc->n_landmarks; ++l) d.l_size[l] = static_cast<float>(desc->landmark_size[l]);
    d.g_agents = desc->n_agents; d.g_landmarks = desc->n_landmarks; d.g_dim_c = desc->dim_c;
    int slot = 0;
    for (int i = 0; i < desc->n_agents; ++i) {
        if (desc->agent_movable[i]) d.g_movable |= 1u << i;
        if (desc->agent_collide[i]) d.g_collide |= 1u << i;
        if (desc->agent_silent[i]) d.g_silent |= 1u << i;
        d.g_slot[i] = desc->agent_silent[i] ? static_cast<int8_t>(-1) : static_cast<int8_t>(slot++);
    }
    for (int l = 0; l < desc->n_landmarks; ++l)
        if (desc->landmark_collide[l]) d.g_lcollide |= 1u << l;
    d.g_comm_rows = slot * desc->dim_c;
    *out = h;
    return MPE_OK;
}

extern "C" int mpe_destroy(mpe_handle h) {
    if (!h) return MPE_ERR_BAD_ARG;
    for (int k = 0; k < 2; ++k) {
        if (h->aux[k]) cudaStreamDestroy(h->aux[k]);
        if (h->ev_join[k]) cudaEventDestroy(h->ev_join[k]);
    }
    if (h->ev_fork) cudaEventDestroy(h->ev_fork);
    delete h;
    return MPE_OK;
}

extern "C" int mpe_num_agents(mpe_handle h) { return h ? h->prog->A : MPE_ERR_BAD_ARG; }
extern "C" int64_t mpe_num_envs(mpe_handle h) { return h ? h->n : static_cast<int64_t>(MPE_ERR_BAD_ARG); }
extern "C" int mpe_obs_dim(mpe_handle h, int i) {
    if (!h || i < 0 || i >= h->prog->A) return MPE_ERR_BAD_ARG;
    return h->prog->scenario == MPE_SCN_CUSTOM ? MPE_ERR_UNSUPPORTED : h->prog->obs_dim[i];
}
extern "C" int mpe_act_dim(mpe_handle h, int i) { return (h && i >= 0 && i < h->prog->A) ? h->prog->act_dim[i] : MPE_ERR_BAD_ARG; }
extern "C" int mpe_num_speakers(mpe_handle h) { return h ? h->prog->NS : MPE_ERR_BAD_ARG; }
extern "C" int mpe_num_goals(mpe_handle h) { return h ? h->prog->G : MPE_ERR_BAD_ARG; }
extern "C" int mpe_info_dim(mpe_handle h) { return h ? h->prog->INFO : MPE_ERR_BAD_ARG; }

extern "C" int64_t mpe_bytes_per_env_step(mpe_handle h) {
    if (!h) return MPE_ERR_BAD_ARG;
    // SURVEY.md 8(d): read agent pos+vel, landmark pos, goal indices, actions; write pos+vel of the movable
    // agents, observations, rewards, speaker comm state, 1 done byte per agent
    const Program *p = h->prog;
    int64_t f = 4 * p->A + 2 * p->L + p->G + p->A + p->NS * p->DIMC - p->unread_state_floats;
    for (int i = 0; i < p->A; ++i) f += p->act_dim[i] + p->obs_dim[i] + (h->desc.agent_movable[i] ? 4 : 0);
    return 4 * f + p->A;
}

// One kernel launch on the handle's device, counted in mpe_kernel_launches.  `pdl` sets programmatic stream
// serialization: the kernel may start while the previous one on the stream is finishing (the step kernels wait for it
// with griddepcontrol.wait before touching global memory).
static int launch_kernel(mpe_handle h, const void *fn, int64_t blocks, int threads, size_t smem, void *stream,
                         void **params, bool pdl, const char *what, unsigned blocks_y = 1) {
    if (blocks > 0x7fffffffLL) return MPE_ERR_BAD_ARG;
    int prev = 0;
    CUDA_TRY(cudaGetDevice(&prev));
    if (prev != h->device) CUDA_TRY(cudaSetDevice(h->device));
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(static_cast<unsigned>(blocks), blocks_y);
    cfg.blockDim = dim3(static_cast<unsigned>(threads));
    cfg.dynamicSmemBytes = smem;
    cfg.stream = static_cast<cudaStream_t>(stream);
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    cudaError_t e = cudaLaunchKernelExC(&cfg, fn, params);
    if (prev != h->device) cudaSetDevice(prev);
    if (e != cudaSuccess) return cuda_fail(e, what);
    __atomic_add_fetch(&g_launches, 1, __ATOMIC_RELAXED);
    return MPE_OK;
}

// Programmatic dependent launch between consecutive step kernels.  MPE_B200_PDL: 0 = off, 1 = release the next grid
// before our stores, 2 = at entry, 3 = once our inputs have arrived (DEFAULT), 4 = implicitly at exit, 5 = as soon as our
// loads are issued
static int pdl_mode() {
    static const int m = [] { const char *e = getenv("MPE_B200_PDL"); return (e && e[0] >= '0' && e[0] <= '5') ? e[0] - '0' : 3; }();
    return m;
}

static int launch(mpe_handle h, int mode, StepArgs &args, void *stream, int64_t begin = 0, int64_t count = -1) {
    if (h->device < 0) return MPE_ERR_NO_DEVICE;
    args.d = h->dev;
    args.n = h->n;
    args.begin = begin;
    args.count = count < 0 ? h->n - begin : count;
    if (h->prog->scenario == MPE_SCN_CUSTOM) {   // generic program: one thread per world, no staging
        if (h->prog->fn[mode] == nullptr) return MPE_ERR_UNSUPPORTED;
        void *params[] = {&args};
        return launch_kernel(h, reinterpret_cast<const void *>(h->prog->fn[mode]), (args.count + 127) / 128, 128, 0, stream,
                             params, false, "cudaLaunchKernelExC(generic)");
    }
    static const int wpb_env = [] { const char *e = getenv("MPE_B200_WPB"); int v = e ? atoi(e) : 0; return (v >= 1 && v <= kMaxWarpsPerBlock) ? v : 0; }();
    static const bool hot_env = [] { const char *e = getenv("MPE_B200_HOT"); return !(e && e[0] == '0'); }();   // 0 = general kernel only
    if (pdl_mode() == 2) args.flags |= kFlagPdlEarly;
    if (pdl_mode() == 3) args.flags |= kFlagPdlAfterLoads;
    if (pdl_mode() == 4) args.flags |= kFlagPdlAtExit;
    if (pdl_mode() == 5) args.flags |= kFlagPdlAfterIssue;
    // one grid of autonomous warps over [sa.begin, sa.begin + sa.count)
    auto launch_grid = [&](KernelFn fn, StepArgs &sa, int max_wpb = kMaxWarpsPerBlock) -> int {
        const int64_t nw = (sa.count + 31) / 32;
        // Warps are autonomous, so the block size only sets scheduling granularity.  While every warp of the batch is
        // resident at once (<= 16 per SM) one warp per block balances the SMs best; mid-size batches use two, large
        // ones four.
        int wpb = wpb_env ? wpb_env : (nw <= 16LL * h->sms ? 1 : (nw <= 64LL * h->sms ? 2 : 4));
        if (wpb > max_warps_per_block(h->prog->smem_bytes)) wpb = max_warps_per_block(h->prog->smem_bytes);
        if (wpb > max_wpb) wpb = max_wpb;
        void *params[] = {&sa};
        return launch_kernel(h, reinterpret_cast<const void *>(fn), (nw + wpb - 1) / wpb, 32 * wpb,
                             static_cast<size_t>(h->prog->smem_bytes) * wpb, stream, params, pdl_mode() != 0,
                             "cudaLaunchKernelExC(step)");
    };
    int rc = MPE_OK;
    // the specialised fused step (mpe_kernel<..., HOT>) takes every whole tile it is eligible for
    bool hot = hot_env && mode == kFusedStep && h->prog->hot_fn != nullptr && args.count >= 32 &&
               !(args.flags & (MPE_FLAG_DISCRETE_ACTION_INPUT | MPE_FLAG_FORCE_DISCRETE_ACTION));
    for (int i = 0; hot && i < h->prog->A; ++i)
        hot = ((reinterpret_cast<uintptr_t>(args.act[i]) + static_cast<uintptr_t>(args.begin) * h->prog->act_dim[i] * 4) & 15u) == 0;
    if (hot) {
        StepArgs ha = args;
        ha.count = args.count / 32 * 32;
        // more tiles than the 128-register kernel keeps resident (16 warps per SM): the 80-register build, if there is one
        static const int dense_env = [] { const char *e = getenv("MPE_B200_DENSE"); return e ? atoi(e) : -1; }();   // 0 never, 1 always
        const bool dense = h->prog->hot_dense_fn != nullptr &&
                           (dense_env == 1 || (dense_env < 0 && ha.count / 32 > 16LL * h->sms));
        rc = dense ? launch_grid(h->prog->hot_dense_fn, ha, 4) : launch_grid(h->prog->hot_fn, ha);
        args.begin += ha.count;
        args.count -= ha.count;
    }
    if (rc == MPE_OK && args.count > 0) rc = launch_grid(h->prog->fn[mode], args);
    return rc;
}

static bool ok16(const void *p) { return p != nullptr && (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
static bool ok8(const void *p) { return p != nullptr && (reinterpret_cast<uintptr_t>(p) & 7u) == 0; }
static bool ok4(const void *p) { return p != nullptr && (reinterpret_cast<uintptr_t>(p) & 3u) == 0; }

static int fill_state(mpe_handle h, StepArgs &a, void *pv, const void *lm, float *comm, const int32_t *goal,
                      bool need_goal = true) {
    const Program *p = h->prog;
    if (!ok16(pv)) return MPE_ERR_BAD_ARG;
    if (p->L > 0 && !ok8(lm)) return MPE_ERR_BAD_ARG;
    if (p->NS * p->DIMC > 0 && !ok4(comm)) return MPE_ERR_BAD_ARG;
    if (need_goal && p->G > 0 && !ok4(goal)) return MPE_ERR_BAD_ARG;
    a.pv = static_cast<float4 *>(pv);
    a.lm = static_cast<const float2 *>(lm);
    a.comm = comm;
    a.goal = goal;
    return MPE_OK;
}

static int fill_outputs(mpe_handle h, StepArgs &a, float *const *obs_n, float *rew, uint8_t *done, float *info) {
    const Program *p = h->prog;
    if (!obs_n || !ok4(rew) || !done) return MPE_ERR_BAD_ARG;
    for (int i = 0; i < p->A; ++i) {
        if (!ok16(obs_n[i])) return MPE_ERR_BAD_ARG;   // observation rows are written as 16-byte stores
        a.obs[i] = obs_n[i];
    }
    a.rew = rew;
    a.done = done;
    a.info = p->INFO > 0 ? info : nullptr;
    return MPE_OK;
}

static int fill_actions(mpe_handle h, StepArgs &a, const float *const *act_n) {
    if (!act_n) return MPE_ERR_BAD_ARG;
    for (int i = 0; i < h->prog->A; ++i) {
        if (!ok4(act_n[i])) return MPE_ERR_BAD_ARG;
        a.act[i] = act_n[i];
    }
    return MPE_OK;
}

// The persistent (multi-step) kernels: one launch covers the whole batch and writes no info
static int fill_persistent(mpe_handle h, StepArgs &a, void *pv, const void *lm, float *comm, const int32_t *goal,
                           float *const *obs_n, float *rew, uint8_t *done, uint32_t flags) {
    int r = fill_state(h, a, pv, lm, comm, goal);
    if (r) return r;
    r = fill_outputs(h, a, obs_n, rew, done, nullptr);
    if (r) return r;
    a.flags = flags;
    a.d = h->dev;
    a.n = h->n;
    a.begin = 0;
    a.count = h->n;
    return MPE_OK;
}

// `warps` warps (one per 32 worlds) in blocks of wpb; dynamic shared memory = fixed bytes + per-warp bytes x wpb
static int launch_persistent(mpe_handle h, const void *fn, int64_t warps, int64_t wpb, size_t fixed_smem, size_t warp_smem,
                             void *args, void *stream, const char *what) {
    void *params[] = {args};
    return launch_kernel(h, fn, (warps + wpb - 1) / wpb, static_cast<int>(32 * wpb), fixed_smem + warp_smem * wpb, stream,
                         params, false, what);
}

extern "C" int mpe_set_action(mpe_handle h, const float *const *act_n, float *u, float *c, uint32_t flags, void *stream) {
    if (!h || !ok8(u)) return MPE_ERR_BAD_ARG;
    if (h->prog->NS * h->prog->DIMC > 0 && !ok4(c)) return MPE_ERR_BAD_ARG;
    StepArgs a{};
    int r = fill_actions(h, a, act_n);
    if (r) return r;
    a.u = reinterpret_cast<float2 *>(u);
    a.c = c;
    a.flags = flags;
    return launch(h, kSetAction, a, stream);
}

extern "C" int mpe_world_step(mpe_handle h, void *pv, const void *lm, float *comm, const float *u, const float *c, void *stream) {
    if (!h || !ok8(u)) return MPE_ERR_BAD_ARG;
    if (h->prog->NS * h->prog->DIMC > 0 && !ok4(c)) return MPE_ERR_BAD_ARG;
    StepArgs a{};
    int r = fill_state(h, a, pv, lm, comm, nullptr, false);
    if (r) return r;
    a.u = reinterpret_cast<float2 *>(const_cast<float *>(u));
    a.c = const_cast<float *>(c);
    return launch(h, kWorldStep, a, stream);
}

extern "C" int mpe_observe(mpe_handle h, const void *pv, const void *lm, const float *comm, const int32_t *goal,
                           float *const *obs_n, float *rew, uint8_t *done, float *info, uint32_t flags, void *stream) {
    if (!h) return MPE_ERR_BAD_ARG;
    if (h->prog->scenario == MPE_SCN_CUSTOM) return MPE_ERR_UNSUPPORTED;
    StepArgs a{};
    int r = fill_state(h, a, const_cast<void *>(pv), lm, const_cast<float *>(comm), goal);
    if (r) return r;
    r = fill_outputs(h, a, obs_n, rew, done, info);
    if (r) return r;
    a.flags = flags;
    return launch(h, kObserve, a, stream);
}

extern "C" int mpe_step(mpe_handle h, void *pv, const void *lm, float *comm, const int32_t *goal,
                        const float *const *act_n, float *const *obs_n, float *rew, uint8_t *done, float *info,
                        uint32_t flags, void *stream) {
    if (!h) return MPE_ERR_BAD_ARG;
    NvtxRange range("mpe_step");
    StepArgs a{};
    int r = fill_state(h, a, pv, lm, comm, goal);
    if (r) return r;
    r = fill_actions(h, a, act_n);
    if (r) return r;
    r = fill_outputs(h, a, obs_n, rew, done, info);
    if (r) return r;
    a.flags = flags;
    return launch(h, kFusedStep, a, stream);
}

extern "C" int mpe_rollout(mpe_handle h, void *pv, const void *lm, float *comm, const int32_t *goal,
                           const float *const *act_seq, int32_t n_steps, float *const *obs_n, float *rew_sum,
                           float *rew_steps, uint8_t *done, uint32_t flags, void *stream) {
    if (!h || n_steps < 0) return MPE_ERR_BAD_ARG;
    if (h->device < 0) return MPE_ERR_NO_DEVICE;
    if (h->prog->scenario == MPE_SCN_CUSTOM || h->prog->rollout_fn == nullptr) return MPE_ERR_UNSUPPORTED;
    if (flags & MPE_FLAG_DISCRETE_ACTION_INPUT) return MPE_ERR_UNSUPPORTED;
    if (rew_steps != nullptr && !ok4(rew_steps)) return MPE_ERR_BAD_ARG;
    NvtxRange range("mpe_rollout");
    RolloutArgs ra{};
    int r = fill_persistent(h, ra.s, pv, lm, comm, goal, obs_n, rew_sum, done, flags);
    if (r) return r;
    r = fill_actions(h, ra.s, act_seq);
    if (r) return r;
    ra.T = n_steps;
    ra.rew_steps = rew_steps;
    const int64_t warps = (h->n + 31) / 32;
    int wpb = warps <= 4LL * h->sms ? 1 : (warps <= 64LL * h->sms ? 2 : 4);
    if (wpb > max_warps_per_block(h->prog->rollout_smem)) wpb = max_warps_per_block(h->prog->rollout_smem);
    return launch_persistent(h, reinterpret_cast<const void *>(h->prog->rollout_fn), warps, wpb, 0, h->prog->rollout_smem, &ra,
                             stream, "cudaLaunchKernelExC(rollout)");
}

extern "C" int mpe_rollout_policy(mpe_handle h, void *pv, const void *lm, float *comm, const int32_t *goal,
                                  const float *const *w1_n, const float *const *b1_n, const float *const *w2_n,
                                  const float *const *b2_n, int32_t hidden, int32_t n_steps, float *const *obs_n,
                                  float *rew_sum, float *rew_steps, float *const *act_record_n, uint8_t *done,
                                  uint32_t flags, void *stream) {
    if (!h || n_steps < 0 || !w1_n || !b1_n || !w2_n || !b2_n) return MPE_ERR_BAD_ARG;
    if (h->device < 0) return MPE_ERR_NO_DEVICE;
    const int k = hidden == 32 ? 0 : (hidden == 64 ? 1 : -1);
    if (k < 0 || h->prog->scenario == MPE_SCN_CUSTOM || h->prog->policy_fn[k] == nullptr) return MPE_ERR_UNSUPPORTED;
    if (flags & (MPE_FLAG_DISCRETE_ACTION_INPUT | MPE_FLAG_FORCE_DISCRETE_ACTION)) return MPE_ERR_UNSUPPORTED;
    if (rew_steps != nullptr && !ok4(rew_steps)) return MPE_ERR_BAD_ARG;
    NvtxRange range("mpe_rollout_policy");
    PolicyArgs pa{};
    int r = fill_persistent(h, pa.s, pv, lm, comm, goal, obs_n, rew_sum, done, flags);
    if (r) return r;
    for (int i = 0; i < h->prog->A; ++i) {
        if (!ok16(w1_n[i]) || !ok16(b1_n[i]) || !ok16(w2_n[i]) || !ok4(b2_n[i])) return MPE_ERR_BAD_ARG;
        pa.w1[i] = w1_n[i]; pa.b1[i] = b1_n[i]; pa.w2[i] = w2_n[i]; pa.b2[i] = b2_n[i];
        pa.act_rec[i] = act_record_n ? act_record_n[i] : nullptr;
        if (pa.act_rec[i] != nullptr && !ok4(pa.act_rec[i])) return MPE_ERR_BAD_ARG;
    }
    pa.T = n_steps;
    pa.rew_steps = rew_steps;
    const int64_t warps = (h->n + 31) / 32;
    const int wpb = warps <= 16LL * h->sms ? 1 : (warps <= 64LL * h->sms ? 2 : 4);
    return launch_persistent(h, reinterpret_cast<const void *>(h->prog->policy_fn[k]), warps, wpb,
                             static_cast<size_t>(h->prog->policy_weight_floats[k]) * 4, h->prog->smem_bytes, &pa, stream,
                             "cudaLaunchKernelExC(rollout_policy)");
}

// The arguments of the six two-hidden-layer rollout entry points, filled by name (several neighbours share a type).
// form: episodes | kind << 1 (kMlpForms).  T is the episode length (n_steps in the single-episode forms); a record the
// form does not have is null.  net_flags and ln_eps are MAPPO's (MlpMappoArgs); forms 6 and 7 (kMlpForms + episodes)
// are the recurrent actor's, whose w[j] hold the shared set's pointer for every agent and gru its MlpGruState; forms 8
// and 9 (kMlpForms + 2 + episodes) MAPPO's actor with critic, the critics' count, weights and value records; forms 10
// and 11 (kMlpForms + 4 + episodes) the same with IPPO's local critics.
struct MlpCall {
    int form;
    MlpGruState gru;
    // per-agent recurrent actors (forms 6 and 7 with separated): W_ih, b_ih, W_hh, b_hh one pointer per agent each (the
    // base and head in w), and the workspace of their fragment images
    bool separated;
    const float *const *gru_w[4];
    void *workspace;
    int64_t workspace_bytes;
    MlpCriticState critic;
    uint32_t net_flags;
    float ln_eps;
    void *pv;
    const void *lm;                   // writable in the episode forms: every episode end redraws them
    float *comm;
    const int32_t *goal;
    const float *const *w[6];         // W1, b1, W2, b2, W3, b3: one pointer per agent each
    int32_t hidden, T, episodes, explore;
    uint64_t explore_seed, explore_epoch, reset_seed, reset_epoch, world_offset;
    float *const *obs_n;
    float *rew, *rew_steps, *logp_steps;
    float *const *act_record_n;
    int32_t *const *act_index_record_n;
    float *const *obs_record_n, *const *final_obs_record_n;
    uint8_t *done;
    uint32_t flags;
    void *stream;
};

static int rollout_policy_mlp(mpe_handle h, const MlpCall &c) {
    static const char *const kName[kMlpForms + 6][2] = {   // the NVTX range, the launch's error context
        {"mpe_rollout_policy_mlp", "cudaLaunchKernelExC(rollout_policy_mlp)"},
        {"mpe_rollout_policy_mlp_episodes", "cudaLaunchKernelExC(rollout_policy_mlp_episodes)"},
        {"mpe_rollout_policy_mlp_categorical", "cudaLaunchKernelExC(rollout_policy_mlp_categorical)"},
        {"mpe_rollout_policy_mlp_categorical_episodes", "cudaLaunchKernelExC(rollout_policy_mlp_categorical_episodes)"},
        {"mpe_rollout_policy_mappo", "cudaLaunchKernelExC(rollout_policy_mappo)"},
        {"mpe_rollout_policy_mappo_episodes", "cudaLaunchKernelExC(rollout_policy_mappo_episodes)"},
        {"mpe_rollout_policy_gru", "cudaLaunchKernelExC(rollout_policy_gru)"},
        {"mpe_rollout_policy_gru_episodes", "cudaLaunchKernelExC(rollout_policy_gru_episodes)"},
        {"mpe_rollout_policy_mappo_critic", "cudaLaunchKernelExC(rollout_policy_mappo_critic)"},
        {"mpe_rollout_policy_mappo_critic_episodes", "cudaLaunchKernelExC(rollout_policy_mappo_critic_episodes)"},
        {"mpe_rollout_policy_mappo_local_critic", "cudaLaunchKernelExC(rollout_policy_mappo_local_critic)"},
        {"mpe_rollout_policy_mappo_local_critic_episodes",
         "cudaLaunchKernelExC(rollout_policy_mappo_local_critic_episodes)"}};
    const bool episodes = c.form & 1, categorical = c.form >= 2, mappo = c.form >= 4;
    const bool gru = c.form == kMlpForms || c.form == kMlpForms + 1, critic = c.form >= kMlpForms + 2;
    const bool local = c.form >= kMlpForms + 4;
    const bool no_weights = !c.w[0] || !c.w[1] || !c.w[2] || !c.w[3] || !c.w[4] || !c.w[5] ||
                            (c.separated && (!c.gru_w[0] || !c.gru_w[1] || !c.gru_w[2] || !c.gru_w[3]));
    // the single-episode forms refuse a negative n_steps and null weight arrays before anything else, the episode forms
    // after the device, program and length checks
    if (!h || (!episodes && (c.T < 0 || no_weights))) return MPE_ERR_BAD_ARG;
    if (h->device < 0) return MPE_ERR_NO_DEVICE;
    const int k = c.hidden == 32 ? 0 : (c.hidden == 64 ? 1 : -1);
    // the per-agent recurrent actors' rollout (hidden width 64 only), else the form's kernel
    const void *const fn = k < 0 ? nullptr
                         : c.separated ? (k == 1 ? h->prog->gru_sep_fn[1 + episodes] : nullptr) : h->prog->mlp[c.form][k].fn;
    if (k < 0 || h->prog->scenario == MPE_SCN_CUSTOM || fn == nullptr) return MPE_ERR_UNSUPPORTED;
    // 1 (shared) or A critics, whose weights must leave room for a warp's tiles next to the actor's.  One shared local
    // critic needs agents that observe alike.
    int critic_cap = 0, critic_floats = 0;
    if (critic) {
        if (c.critic.count != 1 && c.critic.count != h->prog->A) return MPE_ERR_BAD_ARG;
        critic_floats = local ? h->prog->local_critic_floats[c.critic.count == 1 ? 0 : 1]
                              : c.critic.count * h->prog->critic_floats;
        if (local && critic_floats == 0) return MPE_ERR_BAD_ARG;
        critic_cap = (kMlpSmemBytes / 4 - h->prog->mlp_weight_floats[k] - critic_floats) / h->prog->mlp_warp_floats[k];
        if (critic_cap < 1) return MPE_ERR_UNSUPPORTED;
    }
    if (c.flags & (MPE_FLAG_DISCRETE_ACTION_INPUT | MPE_FLAG_FORCE_DISCRETE_ACTION)) return MPE_ERR_UNSUPPORTED;
    // unknown network flags, or an eps that is negative, NaN or infinite
    if (mappo && ((c.net_flags & ~(kMappoFeatureNorm | kMappoTanh)) || !(c.ln_eps >= 0.0f && c.ln_eps <= 3.4e38f)))
        return MPE_ERR_BAD_ARG;
    // records are indexed by the global step e * episode_length + t, an int
    if (episodes && (c.T < 1 || c.episodes < 1 || static_cast<int64_t>(c.T) * c.episodes > 0x7fffffffLL))
        return MPE_ERR_BAD_ARG;
    // the Philox counter word holds (t * A + i) * S + b below the tag bit; t restarts at 0 every episode
    if (c.explore && static_cast<int64_t>(c.T) * h->prog->A * h->prog->mlp_explore_stride > static_cast<int64_t>(kExploreTag))
        return MPE_ERR_BAD_ARG;
    if (no_weights || (c.rew_steps != nullptr && !ok4(c.rew_steps))) return MPE_ERR_BAD_ARG;
    if (gru && ((!c.separated && (!ok4(c.gru.w_ih) || !ok4(c.gru.b_ih) || !ok4(c.gru.w_hh) || !ok4(c.gru.b_hh))) ||
                !ok8(c.gru.h) || (c.gru.h_rec != nullptr && !ok8(c.gru.h_rec))))
        return MPE_ERR_BAD_ARG;
    if (critic) {
        if (!ok4(c.critic.values) || !ok4(c.critic.final_values)) return MPE_ERR_BAD_ARG;
        for (int q = 0; q < c.critic.count; ++q)
            if (!ok4(c.critic.w1[q]) || !ok4(c.critic.b1[q]) || !ok4(c.critic.w2[q]) || !ok4(c.critic.b2[q]) ||
                !ok4(c.critic.w3[q]) || !ok4(c.critic.b3[q]))
                return MPE_ERR_BAD_ARG;
    }
    NvtxRange range(!c.separated ? kName[c.form][0]
                                 : episodes ? "mpe_rollout_policy_gru_separated_episodes" : "mpe_rollout_policy_gru_separated");
    MlpCategoricalRecords cr{};
    if (categorical) {
        if (c.logp_steps != nullptr && !ok4(c.logp_steps)) return MPE_ERR_BAD_ARG;
        cr.logp = c.logp_steps;
        for (int i = 0; i < h->prog->A; ++i) {
            cr.index[i] = c.act_index_record_n ? c.act_index_record_n[i] : nullptr;
            if (cr.index[i] != nullptr && !ok4(cr.index[i])) return MPE_ERR_BAD_ARG;
        }
    }
    MlpEpisodeArgs ea{};
    MlpPolicyArgs &pa = ea.p;
    int r = fill_persistent(h, pa.s, c.pv, c.lm, c.comm, c.goal, c.obs_n, c.rew, c.done, c.flags);
    if (r) return r;
    for (int i = 0; i < h->prog->A; ++i) {
        for (int j = 0; j < 6; ++j)
            if (!ok4(c.w[j][i])) return MPE_ERR_BAD_ARG;
        if (c.separated)
            for (int j = 0; j < 4; ++j)
                if (!ok4(c.gru_w[j][i])) return MPE_ERR_BAD_ARG;
        pa.w1[i] = c.w[0][i]; pa.b1[i] = c.w[1][i]; pa.w2[i] = c.w[2][i]; pa.b2[i] = c.w[3][i]; pa.w3[i] = c.w[4][i]; pa.b3[i] = c.w[5][i];
        pa.act_rec[i] = c.act_record_n ? c.act_record_n[i] : nullptr;
        if (pa.act_rec[i] != nullptr && !ok4(pa.act_rec[i])) return MPE_ERR_BAD_ARG;
        pa.obs_rec[i] = c.obs_record_n ? c.obs_record_n[i] : nullptr;
        if (pa.obs_rec[i] != nullptr && !ok16(pa.obs_rec[i])) return MPE_ERR_BAD_ARG;   // 16-byte tile stores
        ea.final_obs[i] = c.final_obs_record_n ? c.final_obs_record_n[i] : nullptr;
        if (c.final_obs_record_n != nullptr && !ok16(ea.final_obs[i])) return MPE_ERR_BAD_ARG;   // every agent's, or none
    }
    // the fragment images are read by 16-byte bulk copies
    if (c.separated && (!ok16(c.workspace) || c.workspace_bytes < h->prog->gru_sep_image_bytes)) return MPE_ERR_BAD_ARG;
    pa.T = c.T;
    pa.explore = c.explore ? 1 : 0;
    pa.seed = c.explore_seed;
    pa.epoch = c.explore_epoch;
    pa.world_offset = c.world_offset;
    pa.rew_steps = c.rew_steps;
    ea.lm = static_cast<float2 *>(const_cast<void *>(c.lm));
    ea.goal = const_cast<int32_t *>(c.goal);
    ea.episodes = c.episodes;
    ea.reset_seed = c.reset_seed;
    ea.reset_epoch = c.reset_epoch;
    MlpCategoricalArgs ca{pa, cr};
    MlpCategoricalEpisodeArgs cea{ea, cr};
    MlpMappoArgs ma{ca, c.ln_eps, c.net_flags};
    MlpMappoEpisodeArgs mea{cea, c.ln_eps, c.net_flags};
    MlpGruArgs ga{ma, c.gru};
    MlpGruEpisodeArgs gea{mea, c.gru};
    MlpCriticArgs va{ma, c.critic};
    MlpCriticEpisodeArgs vea{mea, c.critic};
    void *const form_args[kMlpForms + 6] = {&pa, &ea, &ca, &cea, &ma, &mea, &ga, &gea, &va, &vea, &va, &vea};
    const float *const images = static_cast<const float *>(c.workspace);
    MlpGruSeparatedArgs sga{ga, images};
    MlpGruSeparatedEpisodeArgs sgea{gea, images};
    int cap = c.separated ? kGruWarps : h->prog->mlp[c.form][k].warps;
    if (critic && critic_cap < cap) cap = critic_cap;   // per-agent critics leave fewer warps than the shared one
    // every block stages all agents' weights once, so blocks are as large as possible while every SM still gets work
    const int64_t warps = (h->n + 31) / 32;
    int64_t wpb = (warps + h->sms - 1) / (h->sms > 0 ? h->sms : 1);
    if (wpb < 1) wpb = 1;
    if (wpb > cap) wpb = cap;
    if (c.separated) {   // every agent's fragment image, then the rollout that restages them turn by turn
        GruImageArgs ia{};
        for (int i = 0; i < h->prog->A; ++i) {
            const float *const *src[10] = {c.w[0], c.w[1], c.w[2], c.w[3], c.gru_w[0], c.gru_w[1], c.gru_w[2], c.gru_w[3],
                                           c.w[4], c.w[5]};
            for (int j = 0; j < 10; ++j) ia.w[j][i] = src[j][i];
        }
        ia.images = static_cast<float *>(c.workspace);
        void *params[] = {&ia};
        int r = launch_kernel(h, h->prog->gru_sep_fn[0], h->prog->A, kGruImageThreads, 0, c.stream, params, false,
                              "cudaLaunchKernelExC(gru_images)");
        if (r) return r;
        return launch_persistent(h, fn, warps, wpb, static_cast<size_t>(4 + h->prog->gru_sep_slot_floats) * 4,
                                 static_cast<size_t>(h->prog->mlp_warp_floats[k]) * 4,
                                 episodes ? static_cast<void *>(&sgea) : static_cast<void *>(&sga), c.stream,
                                 episodes ? "cudaLaunchKernelExC(rollout_policy_gru_separated_episodes)"
                                          : "cudaLaunchKernelExC(rollout_policy_gru_separated)");
    }
    const int weight_floats = gru ? h->prog->gru_weight_floats : h->prog->mlp_weight_floats[k] + critic_floats;
    return launch_persistent(h, fn, warps, wpb, static_cast<size_t>(weight_floats) * 4,
                             static_cast<size_t>(h->prog->mlp_warp_floats[k]) * 4, form_args[c.form], c.stream,
                             kName[c.form][1]);
}

extern "C" int mpe_rollout_policy_mlp(mpe_handle h, void *pv, const void *lm, float *comm, const int32_t *goal,
                                      const float *const *w1_n, const float *const *b1_n, const float *const *w2_n,
                                      const float *const *b2_n, const float *const *w3_n, const float *const *b3_n,
                                      int32_t hidden, int32_t n_steps, int32_t explore, uint64_t explore_seed,
                                      uint64_t explore_epoch, uint64_t world_offset, float *const *obs_n, float *rew_sum,
                                      float *rew_steps, float *const *act_record_n, float *const *obs_record_n,
                                      uint8_t *done, uint32_t flags, void *stream) {
    MlpCall c{};
    c.pv = pv; c.lm = lm; c.comm = comm; c.goal = goal;
    c.w[0] = w1_n; c.w[1] = b1_n; c.w[2] = w2_n; c.w[3] = b2_n; c.w[4] = w3_n; c.w[5] = b3_n;
    c.hidden = hidden; c.explore = explore; c.explore_seed = explore_seed; c.explore_epoch = explore_epoch;
    c.world_offset = world_offset; c.obs_n = obs_n; c.rew_steps = rew_steps; c.obs_record_n = obs_record_n;
    c.done = done; c.flags = flags; c.stream = stream;
    c.form = 0; c.T = n_steps; c.episodes = 1; c.rew = rew_sum; c.act_record_n = act_record_n;
    return rollout_policy_mlp(h, c);
}

extern "C" int mpe_rollout_policy_mlp_episodes(mpe_handle h, void *pv, void *lm, float *comm, int32_t *goal,
                                               const float *const *w1_n, const float *const *b1_n, const float *const *w2_n,
                                               const float *const *b2_n, const float *const *w3_n, const float *const *b3_n,
                                               int32_t hidden, int32_t episode_length, int32_t n_episodes, int32_t explore,
                                               uint64_t explore_seed, uint64_t explore_epoch, uint64_t reset_seed,
                                               uint64_t reset_epoch, uint64_t world_offset, float *const *obs_n, float *ep_rew,
                                               float *rew_steps, float *const *act_record_n, float *const *obs_record_n,
                                               float *const *final_obs_record_n, uint8_t *done, uint32_t flags, void *stream) {
    MlpCall c{};
    c.pv = pv; c.lm = lm; c.comm = comm; c.goal = goal;
    c.w[0] = w1_n; c.w[1] = b1_n; c.w[2] = w2_n; c.w[3] = b2_n; c.w[4] = w3_n; c.w[5] = b3_n;
    c.hidden = hidden; c.explore = explore; c.explore_seed = explore_seed; c.explore_epoch = explore_epoch;
    c.world_offset = world_offset; c.obs_n = obs_n; c.rew_steps = rew_steps; c.obs_record_n = obs_record_n;
    c.done = done; c.flags = flags; c.stream = stream;
    c.form = 1; c.T = episode_length; c.episodes = n_episodes; c.rew = ep_rew; c.act_record_n = act_record_n;
    c.reset_seed = reset_seed; c.reset_epoch = reset_epoch; c.final_obs_record_n = final_obs_record_n;
    return rollout_policy_mlp(h, c);
}

extern "C" int mpe_rollout_policy_mlp_categorical(mpe_handle h, void *pv, const void *lm, float *comm, const int32_t *goal,
                                                  const float *const *w1_n, const float *const *b1_n,
                                                  const float *const *w2_n, const float *const *b2_n,
                                                  const float *const *w3_n, const float *const *b3_n, int32_t hidden,
                                                  int32_t n_steps, int32_t explore, uint64_t explore_seed,
                                                  uint64_t explore_epoch, uint64_t world_offset, float *const *obs_n,
                                                  float *rew_sum, float *rew_steps, float *logp_steps,
                                                  int32_t *const *act_index_record_n, float *const *obs_record_n,
                                                  uint8_t *done, uint32_t flags, void *stream) {
    MlpCall c{};
    c.pv = pv; c.lm = lm; c.comm = comm; c.goal = goal;
    c.w[0] = w1_n; c.w[1] = b1_n; c.w[2] = w2_n; c.w[3] = b2_n; c.w[4] = w3_n; c.w[5] = b3_n;
    c.hidden = hidden; c.explore = explore; c.explore_seed = explore_seed; c.explore_epoch = explore_epoch;
    c.world_offset = world_offset; c.obs_n = obs_n; c.rew_steps = rew_steps; c.obs_record_n = obs_record_n;
    c.done = done; c.flags = flags; c.stream = stream;
    c.form = 2; c.T = n_steps; c.episodes = 1; c.rew = rew_sum;
    c.logp_steps = logp_steps; c.act_index_record_n = act_index_record_n;
    return rollout_policy_mlp(h, c);
}

extern "C" int mpe_rollout_policy_mlp_categorical_episodes(
    mpe_handle h, void *pv, void *lm, float *comm, int32_t *goal, const float *const *w1_n, const float *const *b1_n,
    const float *const *w2_n, const float *const *b2_n, const float *const *w3_n, const float *const *b3_n, int32_t hidden,
    int32_t episode_length, int32_t n_episodes, int32_t explore, uint64_t explore_seed, uint64_t explore_epoch,
    uint64_t reset_seed, uint64_t reset_epoch, uint64_t world_offset, float *const *obs_n, float *ep_rew, float *rew_steps,
    float *logp_steps, int32_t *const *act_index_record_n, float *const *obs_record_n, float *const *final_obs_record_n,
    uint8_t *done, uint32_t flags, void *stream) {
    MlpCall c{};
    c.pv = pv; c.lm = lm; c.comm = comm; c.goal = goal;
    c.w[0] = w1_n; c.w[1] = b1_n; c.w[2] = w2_n; c.w[3] = b2_n; c.w[4] = w3_n; c.w[5] = b3_n;
    c.hidden = hidden; c.explore = explore; c.explore_seed = explore_seed; c.explore_epoch = explore_epoch;
    c.world_offset = world_offset; c.obs_n = obs_n; c.rew_steps = rew_steps; c.obs_record_n = obs_record_n;
    c.done = done; c.flags = flags; c.stream = stream;
    c.form = 3; c.T = episode_length; c.episodes = n_episodes; c.rew = ep_rew;
    c.logp_steps = logp_steps; c.act_index_record_n = act_index_record_n;
    c.reset_seed = reset_seed; c.reset_epoch = reset_epoch; c.final_obs_record_n = final_obs_record_n;
    return rollout_policy_mlp(h, c);
}

extern "C" int mpe_rollout_policy_mappo(mpe_handle h, void *pv, const void *lm, float *comm, const int32_t *goal,
                                        const float *const *w1_n, const float *const *b1_n, const float *const *w2_n,
                                        const float *const *b2_n, const float *const *w3_n, const float *const *b3_n,
                                        int32_t hidden, int32_t n_steps, int32_t explore, uint64_t explore_seed,
                                        uint64_t explore_epoch, uint64_t world_offset, float *const *obs_n, float *rew_sum,
                                        float *rew_steps, float *logp_steps, int32_t *const *act_index_record_n,
                                        float *const *obs_record_n, uint32_t net_flags, float ln_eps, uint8_t *done,
                                        uint32_t flags, void *stream) {
    MlpCall c{};
    c.pv = pv; c.lm = lm; c.comm = comm; c.goal = goal;
    c.w[0] = w1_n; c.w[1] = b1_n; c.w[2] = w2_n; c.w[3] = b2_n; c.w[4] = w3_n; c.w[5] = b3_n;
    c.hidden = hidden; c.explore = explore; c.explore_seed = explore_seed; c.explore_epoch = explore_epoch;
    c.world_offset = world_offset; c.obs_n = obs_n; c.rew_steps = rew_steps; c.obs_record_n = obs_record_n;
    c.done = done; c.flags = flags; c.stream = stream;
    c.form = 4; c.T = n_steps; c.episodes = 1; c.rew = rew_sum;
    c.logp_steps = logp_steps; c.act_index_record_n = act_index_record_n;
    c.net_flags = net_flags; c.ln_eps = ln_eps;
    return rollout_policy_mlp(h, c);
}

extern "C" int mpe_rollout_policy_mappo_episodes(
    mpe_handle h, void *pv, void *lm, float *comm, int32_t *goal, const float *const *w1_n, const float *const *b1_n,
    const float *const *w2_n, const float *const *b2_n, const float *const *w3_n, const float *const *b3_n, int32_t hidden,
    int32_t episode_length, int32_t n_episodes, int32_t explore, uint64_t explore_seed, uint64_t explore_epoch,
    uint64_t reset_seed, uint64_t reset_epoch, uint64_t world_offset, float *const *obs_n, float *ep_rew, float *rew_steps,
    float *logp_steps, int32_t *const *act_index_record_n, float *const *obs_record_n, float *const *final_obs_record_n,
    uint32_t net_flags, float ln_eps, uint8_t *done, uint32_t flags, void *stream) {
    MlpCall c{};
    c.pv = pv; c.lm = lm; c.comm = comm; c.goal = goal;
    c.w[0] = w1_n; c.w[1] = b1_n; c.w[2] = w2_n; c.w[3] = b2_n; c.w[4] = w3_n; c.w[5] = b3_n;
    c.hidden = hidden; c.explore = explore; c.explore_seed = explore_seed; c.explore_epoch = explore_epoch;
    c.world_offset = world_offset; c.obs_n = obs_n; c.rew_steps = rew_steps; c.obs_record_n = obs_record_n;
    c.done = done; c.flags = flags; c.stream = stream;
    c.form = 5; c.T = episode_length; c.episodes = n_episodes; c.rew = ep_rew;
    c.logp_steps = logp_steps; c.act_index_record_n = act_index_record_n;
    c.reset_seed = reset_seed; c.reset_epoch = reset_epoch; c.final_obs_record_n = final_obs_record_n;
    c.net_flags = net_flags; c.ln_eps = ln_eps;
    return rollout_policy_mlp(h, c);
}

// The recurrent actor's weight set (W1, b1, W2, b2, W_ih, b_ih, W_hh, b_hh, W3, b3) -> every agent's base and head
// pointers and c.gru; a null weight leaves c.w null, which the launcher refuses as MAPPO's null weight arrays
static int rollout_policy_gru(mpe_handle h, MlpCall &c, const float *const (&wt)[10], float *rnn_state,
                              float *rnn_state_record) {
    const float *per_agent[6][kMaxA];
    bool all = true;
    for (int j = 0; j < 10; ++j) all = all && wt[j] != nullptr;
    static const int kBaseHead[6] = {0, 1, 2, 3, 8, 9};
    for (int j = 0; j < 6; ++j) {
        for (int i = 0; i < kMaxA; ++i) per_agent[j][i] = wt[kBaseHead[j]];
        c.w[j] = all ? per_agent[j] : nullptr;
    }
    c.gru = MlpGruState{wt[4], wt[5], wt[6], wt[7], rnn_state, rnn_state_record};
    return rollout_policy_mlp(h, c);
}

extern "C" int mpe_rollout_policy_gru(mpe_handle h, void *pv, const void *lm, float *comm, const int32_t *goal,
                                      const float *w1, const float *b1, const float *w2, const float *b2,
                                      const float *w_ih, const float *b_ih, const float *w_hh, const float *b_hh,
                                      const float *w3, const float *b3, int32_t hidden, int32_t n_steps, int32_t explore,
                                      uint64_t explore_seed, uint64_t explore_epoch, uint64_t world_offset,
                                      float *const *obs_n, float *rew_sum, float *rew_steps, float *logp_steps,
                                      int32_t *const *act_index_record_n, float *const *obs_record_n, float *rnn_state,
                                      float *rnn_state_record, uint32_t net_flags, float ln_eps, uint8_t *done,
                                      uint32_t flags, void *stream) {
    MlpCall c{};
    c.pv = pv; c.lm = lm; c.comm = comm; c.goal = goal;
    c.hidden = hidden; c.explore = explore; c.explore_seed = explore_seed; c.explore_epoch = explore_epoch;
    c.world_offset = world_offset; c.obs_n = obs_n; c.rew_steps = rew_steps; c.obs_record_n = obs_record_n;
    c.done = done; c.flags = flags; c.stream = stream;
    c.form = kMlpForms; c.T = n_steps; c.episodes = 1; c.rew = rew_sum;
    c.logp_steps = logp_steps; c.act_index_record_n = act_index_record_n;
    c.net_flags = net_flags; c.ln_eps = ln_eps;
    return rollout_policy_gru(h, c, {w1, b1, w2, b2, w_ih, b_ih, w_hh, b_hh, w3, b3}, rnn_state, rnn_state_record);
}

extern "C" int mpe_rollout_policy_gru_episodes(
    mpe_handle h, void *pv, void *lm, float *comm, int32_t *goal, const float *w1, const float *b1, const float *w2,
    const float *b2, const float *w_ih, const float *b_ih, const float *w_hh, const float *b_hh, const float *w3,
    const float *b3, int32_t hidden, int32_t episode_length, int32_t n_episodes, int32_t explore, uint64_t explore_seed,
    uint64_t explore_epoch, uint64_t reset_seed, uint64_t reset_epoch, uint64_t world_offset, float *const *obs_n,
    float *ep_rew, float *rew_steps, float *logp_steps, int32_t *const *act_index_record_n, float *const *obs_record_n,
    float *const *final_obs_record_n, float *rnn_state, float *rnn_state_record, uint32_t net_flags, float ln_eps,
    uint8_t *done, uint32_t flags, void *stream) {
    MlpCall c{};
    c.pv = pv; c.lm = lm; c.comm = comm; c.goal = goal;
    c.hidden = hidden; c.explore = explore; c.explore_seed = explore_seed; c.explore_epoch = explore_epoch;
    c.world_offset = world_offset; c.obs_n = obs_n; c.rew_steps = rew_steps; c.obs_record_n = obs_record_n;
    c.done = done; c.flags = flags; c.stream = stream;
    c.form = kMlpForms + 1; c.T = episode_length; c.episodes = n_episodes; c.rew = ep_rew;
    c.logp_steps = logp_steps; c.act_index_record_n = act_index_record_n;
    c.reset_seed = reset_seed; c.reset_epoch = reset_epoch; c.final_obs_record_n = final_obs_record_n;
    c.net_flags = net_flags; c.ln_eps = ln_eps;
    return rollout_policy_gru(h, c, {w1, b1, w2, b2, w_ih, b_ih, w_hh, b_hh, w3, b3}, rnn_state, rnn_state_record);
}

// Per-agent recurrent actors: the ten per-agent weight arrays -> c.w (base and head) and c.gru_w, and the workspace
static int rollout_policy_gru_separated(mpe_handle h, MlpCall &c, const float *const *const (&wt)[10], float *rnn_state,
                                        float *rnn_state_record, void *workspace, int64_t workspace_bytes) {
    static const int kBaseHead[6] = {0, 1, 2, 3, 8, 9};
    for (int j = 0; j < 6; ++j) c.w[j] = wt[kBaseHead[j]];
    for (int j = 0; j < 4; ++j) c.gru_w[j] = wt[4 + j];
    c.separated = true;
    c.gru = MlpGruState{nullptr, nullptr, nullptr, nullptr, rnn_state, rnn_state_record};
    c.workspace = workspace;
    c.workspace_bytes = workspace_bytes;
    return rollout_policy_mlp(h, c);
}

extern "C" int mpe_rollout_policy_gru_separated(
    mpe_handle h, void *pv, const void *lm, float *comm, const int32_t *goal, const float *const *w1_n,
    const float *const *b1_n, const float *const *w2_n, const float *const *b2_n, const float *const *w_ih_n,
    const float *const *b_ih_n, const float *const *w_hh_n, const float *const *b_hh_n, const float *const *w3_n,
    const float *const *b3_n, int32_t hidden, int32_t n_steps, int32_t explore, uint64_t explore_seed,
    uint64_t explore_epoch, uint64_t world_offset, float *const *obs_n, float *rew_sum, float *rew_steps, float *logp_steps,
    int32_t *const *act_index_record_n, float *const *obs_record_n, float *rnn_state, float *rnn_state_record,
    void *workspace, int64_t workspace_bytes, uint32_t net_flags, float ln_eps, uint8_t *done, uint32_t flags,
    void *stream) {
    MlpCall c{};
    c.pv = pv; c.lm = lm; c.comm = comm; c.goal = goal;
    c.hidden = hidden; c.explore = explore; c.explore_seed = explore_seed; c.explore_epoch = explore_epoch;
    c.world_offset = world_offset; c.obs_n = obs_n; c.rew_steps = rew_steps; c.obs_record_n = obs_record_n;
    c.done = done; c.flags = flags; c.stream = stream;
    c.form = kMlpForms; c.T = n_steps; c.episodes = 1; c.rew = rew_sum;
    c.logp_steps = logp_steps; c.act_index_record_n = act_index_record_n;
    c.net_flags = net_flags; c.ln_eps = ln_eps;
    return rollout_policy_gru_separated(h, c, {w1_n, b1_n, w2_n, b2_n, w_ih_n, b_ih_n, w_hh_n, b_hh_n, w3_n, b3_n},
                                        rnn_state, rnn_state_record, workspace, workspace_bytes);
}

extern "C" int mpe_rollout_policy_gru_separated_episodes(
    mpe_handle h, void *pv, void *lm, float *comm, int32_t *goal, const float *const *w1_n, const float *const *b1_n,
    const float *const *w2_n, const float *const *b2_n, const float *const *w_ih_n, const float *const *b_ih_n,
    const float *const *w_hh_n, const float *const *b_hh_n, const float *const *w3_n, const float *const *b3_n,
    int32_t hidden, int32_t episode_length, int32_t n_episodes, int32_t explore, uint64_t explore_seed,
    uint64_t explore_epoch, uint64_t reset_seed, uint64_t reset_epoch, uint64_t world_offset, float *const *obs_n,
    float *ep_rew, float *rew_steps, float *logp_steps, int32_t *const *act_index_record_n, float *const *obs_record_n,
    float *const *final_obs_record_n, float *rnn_state, float *rnn_state_record, void *workspace, int64_t workspace_bytes,
    uint32_t net_flags, float ln_eps, uint8_t *done, uint32_t flags, void *stream) {
    MlpCall c{};
    c.pv = pv; c.lm = lm; c.comm = comm; c.goal = goal;
    c.hidden = hidden; c.explore = explore; c.explore_seed = explore_seed; c.explore_epoch = explore_epoch;
    c.world_offset = world_offset; c.obs_n = obs_n; c.rew_steps = rew_steps; c.obs_record_n = obs_record_n;
    c.done = done; c.flags = flags; c.stream = stream;
    c.form = kMlpForms + 1; c.T = episode_length; c.episodes = n_episodes; c.rew = ep_rew;
    c.logp_steps = logp_steps; c.act_index_record_n = act_index_record_n;
    c.reset_seed = reset_seed; c.reset_epoch = reset_epoch; c.final_obs_record_n = final_obs_record_n;
    c.net_flags = net_flags; c.ln_eps = ln_eps;
    return rollout_policy_gru_separated(h, c, {w1_n, b1_n, w2_n, b2_n, w_ih_n, b_ih_n, w_hh_n, b_hh_n, w3_n, b3_n},
                                        rnn_state, rnn_state_record, workspace, workspace_bytes);
}

extern "C" int64_t mpe_rollout_policy_gru_separated_workspace_bytes(mpe_handle h) {
    if (!h) return MPE_ERR_BAD_ARG;
    if (h->prog->scenario == MPE_SCN_CUSTOM || h->prog->gru_sep_fn[0] == nullptr) return MPE_ERR_UNSUPPORTED;
    return h->prog->gru_sep_image_bytes;
}

// The critics' six weight arrays (W1, b1, W2, b2, W3, b3: critic_count pointers each) and value records -> c.critic
static int rollout_policy_critic(mpe_handle h, MlpCall &c, int32_t critic_count, const float *const *const (&cw)[6],
                                 float *values, float *final_values) {
    c.critic.count = critic_count;
    c.critic.values = values;
    c.critic.final_values = final_values;
    const float **dst[6] = {c.critic.w1, c.critic.b1, c.critic.w2, c.critic.b2, c.critic.w3, c.critic.b3};
    for (int j = 0; j < 6; ++j)
        for (int q = 0; q < critic_count && q < kMaxA; ++q) dst[j][q] = cw[j] ? cw[j][q] : nullptr;
    return rollout_policy_mlp(h, c);
}

extern "C" int mpe_rollout_policy_mappo_critic(
    mpe_handle h, void *pv, const void *lm, float *comm, const int32_t *goal, const float *const *w1_n,
    const float *const *b1_n, const float *const *w2_n, const float *const *b2_n, const float *const *w3_n,
    const float *const *b3_n, int32_t hidden, int32_t n_steps, int32_t explore, uint64_t explore_seed,
    uint64_t explore_epoch, uint64_t world_offset, float *const *obs_n, float *rew_sum, float *rew_steps, float *logp_steps,
    int32_t *const *act_index_record_n, float *const *obs_record_n, uint32_t net_flags, float ln_eps, int32_t critic_count,
    const float *const *cw1, const float *const *cb1, const float *const *cw2, const float *const *cb2,
    const float *const *cw3, const float *const *cb3, float *values, float *final_values, uint8_t *done, uint32_t flags,
    void *stream) {
    MlpCall c{};
    c.pv = pv; c.lm = lm; c.comm = comm; c.goal = goal;
    c.w[0] = w1_n; c.w[1] = b1_n; c.w[2] = w2_n; c.w[3] = b2_n; c.w[4] = w3_n; c.w[5] = b3_n;
    c.hidden = hidden; c.explore = explore; c.explore_seed = explore_seed; c.explore_epoch = explore_epoch;
    c.world_offset = world_offset; c.obs_n = obs_n; c.rew_steps = rew_steps; c.obs_record_n = obs_record_n;
    c.done = done; c.flags = flags; c.stream = stream;
    c.form = kMlpForms + 2; c.T = n_steps; c.episodes = 1; c.rew = rew_sum;
    c.logp_steps = logp_steps; c.act_index_record_n = act_index_record_n;
    c.net_flags = net_flags; c.ln_eps = ln_eps;
    return rollout_policy_critic(h, c, critic_count, {cw1, cb1, cw2, cb2, cw3, cb3}, values, final_values);
}

extern "C" int mpe_rollout_policy_mappo_critic_episodes(
    mpe_handle h, void *pv, void *lm, float *comm, int32_t *goal, const float *const *w1_n, const float *const *b1_n,
    const float *const *w2_n, const float *const *b2_n, const float *const *w3_n, const float *const *b3_n, int32_t hidden,
    int32_t episode_length, int32_t n_episodes, int32_t explore, uint64_t explore_seed, uint64_t explore_epoch,
    uint64_t reset_seed, uint64_t reset_epoch, uint64_t world_offset, float *const *obs_n, float *ep_rew, float *rew_steps,
    float *logp_steps, int32_t *const *act_index_record_n, float *const *obs_record_n, float *const *final_obs_record_n,
    uint32_t net_flags, float ln_eps, int32_t critic_count, const float *const *cw1, const float *const *cb1,
    const float *const *cw2, const float *const *cb2, const float *const *cw3, const float *const *cb3, float *values,
    float *final_values, uint8_t *done, uint32_t flags, void *stream) {
    MlpCall c{};
    c.pv = pv; c.lm = lm; c.comm = comm; c.goal = goal;
    c.w[0] = w1_n; c.w[1] = b1_n; c.w[2] = w2_n; c.w[3] = b2_n; c.w[4] = w3_n; c.w[5] = b3_n;
    c.hidden = hidden; c.explore = explore; c.explore_seed = explore_seed; c.explore_epoch = explore_epoch;
    c.world_offset = world_offset; c.obs_n = obs_n; c.rew_steps = rew_steps; c.obs_record_n = obs_record_n;
    c.done = done; c.flags = flags; c.stream = stream;
    c.form = kMlpForms + 3; c.T = episode_length; c.episodes = n_episodes; c.rew = ep_rew;
    c.logp_steps = logp_steps; c.act_index_record_n = act_index_record_n;
    c.reset_seed = reset_seed; c.reset_epoch = reset_epoch; c.final_obs_record_n = final_obs_record_n;
    c.net_flags = net_flags; c.ln_eps = ln_eps;
    return rollout_policy_critic(h, c, critic_count, {cw1, cb1, cw2, cb2, cw3, cb3}, values, final_values);
}

extern "C" int mpe_rollout_policy_mappo_local_critic(
    mpe_handle h, void *pv, const void *lm, float *comm, const int32_t *goal, const float *const *w1_n,
    const float *const *b1_n, const float *const *w2_n, const float *const *b2_n, const float *const *w3_n,
    const float *const *b3_n, int32_t hidden, int32_t n_steps, int32_t explore, uint64_t explore_seed,
    uint64_t explore_epoch, uint64_t world_offset, float *const *obs_n, float *rew_sum, float *rew_steps, float *logp_steps,
    int32_t *const *act_index_record_n, float *const *obs_record_n, uint32_t net_flags, float ln_eps, int32_t critic_count,
    const float *const *cw1, const float *const *cb1, const float *const *cw2, const float *const *cb2,
    const float *const *cw3, const float *const *cb3, float *values, float *final_values, uint8_t *done, uint32_t flags,
    void *stream) {
    MlpCall c{};
    c.pv = pv; c.lm = lm; c.comm = comm; c.goal = goal;
    c.w[0] = w1_n; c.w[1] = b1_n; c.w[2] = w2_n; c.w[3] = b2_n; c.w[4] = w3_n; c.w[5] = b3_n;
    c.hidden = hidden; c.explore = explore; c.explore_seed = explore_seed; c.explore_epoch = explore_epoch;
    c.world_offset = world_offset; c.obs_n = obs_n; c.rew_steps = rew_steps; c.obs_record_n = obs_record_n;
    c.done = done; c.flags = flags; c.stream = stream;
    c.form = kMlpForms + 4; c.T = n_steps; c.episodes = 1; c.rew = rew_sum;
    c.logp_steps = logp_steps; c.act_index_record_n = act_index_record_n;
    c.net_flags = net_flags; c.ln_eps = ln_eps;
    return rollout_policy_critic(h, c, critic_count, {cw1, cb1, cw2, cb2, cw3, cb3}, values, final_values);
}

extern "C" int mpe_rollout_policy_mappo_local_critic_episodes(
    mpe_handle h, void *pv, void *lm, float *comm, int32_t *goal, const float *const *w1_n, const float *const *b1_n,
    const float *const *w2_n, const float *const *b2_n, const float *const *w3_n, const float *const *b3_n, int32_t hidden,
    int32_t episode_length, int32_t n_episodes, int32_t explore, uint64_t explore_seed, uint64_t explore_epoch,
    uint64_t reset_seed, uint64_t reset_epoch, uint64_t world_offset, float *const *obs_n, float *ep_rew, float *rew_steps,
    float *logp_steps, int32_t *const *act_index_record_n, float *const *obs_record_n, float *const *final_obs_record_n,
    uint32_t net_flags, float ln_eps, int32_t critic_count, const float *const *cw1, const float *const *cb1,
    const float *const *cw2, const float *const *cb2, const float *const *cw3, const float *const *cb3, float *values,
    float *final_values, uint8_t *done, uint32_t flags, void *stream) {
    MlpCall c{};
    c.pv = pv; c.lm = lm; c.comm = comm; c.goal = goal;
    c.w[0] = w1_n; c.w[1] = b1_n; c.w[2] = w2_n; c.w[3] = b2_n; c.w[4] = w3_n; c.w[5] = b3_n;
    c.hidden = hidden; c.explore = explore; c.explore_seed = explore_seed; c.explore_epoch = explore_epoch;
    c.world_offset = world_offset; c.obs_n = obs_n; c.rew_steps = rew_steps; c.obs_record_n = obs_record_n;
    c.done = done; c.flags = flags; c.stream = stream;
    c.form = kMlpForms + 5; c.T = episode_length; c.episodes = n_episodes; c.rew = ep_rew;
    c.logp_steps = logp_steps; c.act_index_record_n = act_index_record_n;
    c.reset_seed = reset_seed; c.reset_epoch = reset_epoch; c.final_obs_record_n = final_obs_record_n;
    c.net_flags = net_flags; c.ln_eps = ln_eps;
    return rollout_policy_critic(h, c, critic_count, {cw1, cb1, cw2, cb2, cw3, cb3}, values, final_values);
}

// The checks of the recurrent critics' entry points, in their documented order, and RCriticArgs but for the weights.
// fn: the program's kernel; weights_ok: every weight pointer non-null and 4-byte aligned.
static int rcritic_args(mpe_handle h, const void *fn, const float *const *obs_record_n, const float *const *final_obs_n,
                        int32_t n_steps, int32_t episode_length, bool weights_ok, float *rnn_state,
                        float *rnn_state_record, float *values, float *final_values, uint32_t net_flags, float ln_eps,
                        RCriticArgs &a) {
    if (!h || n_steps < 0) return MPE_ERR_BAD_ARG;
    if (h->device < 0) return MPE_ERR_NO_DEVICE;
    const Program *p = h->prog;
    if (p->scenario == MPE_SCN_CUSTOM || fn == nullptr) return MPE_ERR_UNSUPPORTED;
    if (episode_length < 0 || (episode_length > 0 && (n_steps < 1 || n_steps % episode_length != 0)))
        return MPE_ERR_BAD_ARG;
    // unknown network flags, or an eps that is negative, NaN or infinite
    if ((net_flags & ~(kMappoFeatureNorm | kMappoTanh)) || !(ln_eps >= 0.0f && ln_eps <= 3.4e38f)) return MPE_ERR_BAD_ARG;
    if (!weights_ok) return MPE_ERR_BAD_ARG;
    if (!ok8(rnn_state) || (rnn_state_record != nullptr && !ok8(rnn_state_record)) || !ok4(final_values) || !final_obs_n)
        return MPE_ERR_BAD_ARG;
    if (n_steps > 0 && (!ok4(values) || !obs_record_n)) return MPE_ERR_BAD_ARG;
    for (int i = 0; i < p->A; ++i) {
        if (!ok4(final_obs_n[i]) || (n_steps > 0 && !ok4(obs_record_n[i]))) return MPE_ERR_BAD_ARG;
        a.obs[i] = n_steps > 0 ? obs_record_n[i] : nullptr;
        a.final_obs[i] = final_obs_n[i];
    }
    a.h = rnn_state; a.h_rec = rnn_state_record; a.values = values; a.final_values = final_values;
    a.n = h->n; a.T = n_steps; a.L = episode_length;
    a.net_flags = net_flags; a.ln_eps = ln_eps;
    return MPE_OK;
}

// one warp per 16 worlds, blocks_y critics, weight_floats of weights in shared memory
static int launch_rcritic(mpe_handle h, const void *fn, void *args, unsigned blocks_y, int weight_floats, void *stream,
                          const char *what) {
    const int64_t warps = (h->n + 15) / 16;
    int64_t wpb = (warps + h->sms - 1) / (h->sms > 0 ? h->sms : 1);
    if (wpb < 1) wpb = 1;
    if (wpb > kRCriticWarps) wpb = kRCriticWarps;
    void *params[] = {args};
    return launch_kernel(h, fn, (warps + wpb - 1) / wpb, static_cast<int>(32 * wpb),
                         static_cast<size_t>(weight_floats) * 4, stream, params, false, what, blocks_y);
}

extern "C" int mpe_critic_gru(mpe_handle h, const float *const *obs_record_n, const float *const *final_obs_n,
                              int32_t n_steps, int32_t episode_length, const float *w1, const float *b1, const float *w2,
                              const float *b2, const float *w_ih, const float *b_ih, const float *w_hh, const float *b_hh,
                              const float *w3, const float *b3, float *rnn_state, float *rnn_state_record, float *values,
                              float *final_values, uint32_t net_flags, float ln_eps, void *stream) {
    const float *const wt[10] = {w1, b1, w2, b2, w_ih, b_ih, w_hh, b_hh, w3, b3};
    bool weights_ok = true;
    for (int j = 0; j < 10; ++j) weights_ok = weights_ok && ok4(wt[j]);
    RCriticArgs a{};
    int r = rcritic_args(h, h ? h->prog->critic_gru_fn : nullptr, obs_record_n, final_obs_n, n_steps, episode_length,
                         weights_ok, rnn_state, rnn_state_record, values, final_values, net_flags, ln_eps, a);
    if (r) return r;
    a.w1 = w1; a.b1 = b1; a.w2 = w2; a.b2 = b2; a.w_ih = w_ih; a.b_ih = b_ih; a.w_hh = w_hh; a.b_hh = b_hh;
    a.w3 = w3; a.b3 = b3;
    NvtxRange range("mpe_critic_gru");
    return launch_rcritic(h, h->prog->critic_gru_fn, &a, 1, h->prog->critic_gru_floats, stream,
                          "cudaLaunchKernelExC(critic_gru)");
}

extern "C" int mpe_critic_gru_local(mpe_handle h, const float *const *obs_record_n, const float *const *final_obs_n,
                                    int32_t n_steps, int32_t episode_length, const float *w1, const float *b1,
                                    const float *w2, const float *b2, const float *w_ih, const float *b_ih,
                                    const float *w_hh, const float *b_hh, const float *w3, const float *b3,
                                    float *rnn_state, float *rnn_state_record, float *values, float *final_values,
                                    uint32_t net_flags, float ln_eps, void *stream) {
    const float *const wt[10] = {w1, b1, w2, b2, w_ih, b_ih, w_hh, b_hh, w3, b3};
    bool weights_ok = true;
    for (int j = 0; j < 10; ++j) weights_ok = weights_ok && ok4(wt[j]);
    RCriticArgs a{};
    int r = rcritic_args(h, h ? h->prog->critic_gru_local_fn : nullptr, obs_record_n, final_obs_n, n_steps,
                         episode_length, weights_ok, rnn_state, rnn_state_record, values, final_values, net_flags, ln_eps,
                         a);
    if (r) return r;
    a.w1 = w1; a.b1 = b1; a.w2 = w2; a.b2 = b2; a.w_ih = w_ih; a.b_ih = b_ih; a.w_hh = w_hh; a.b_hh = b_hh;
    a.w3 = w3; a.b3 = b3;
    NvtxRange range("mpe_critic_gru_local");
    return launch_rcritic(h, h->prog->critic_gru_local_fn, &a, static_cast<unsigned>(h->prog->A),
                          h->prog->critic_gru_local_floats, stream, "cudaLaunchKernelExC(critic_gru_local)");
}

extern "C" int mpe_critic_gru_separated(mpe_handle h, const float *const *obs_record_n, const float *const *final_obs_n,
                                        int32_t n_steps, int32_t episode_length, const float *const *w1_n,
                                        const float *const *b1_n, const float *const *w2_n, const float *const *b2_n,
                                        const float *const *w_ih_n, const float *const *b_ih_n,
                                        const float *const *w_hh_n, const float *const *b_hh_n,
                                        const float *const *w3_n, const float *const *b3_n, float *rnn_state,
                                        float *rnn_state_record, float *values, float *final_values, uint32_t net_flags,
                                        float ln_eps, void *stream) {
    const float *const *const wt[10] = {w1_n, b1_n, w2_n, b2_n, w_ih_n, b_ih_n, w_hh_n, b_hh_n, w3_n, b3_n};
    RCriticSeparatedArgs sa{};
    bool weights_ok = h != nullptr;
    for (int j = 0; j < 10 && weights_ok; ++j) {
        weights_ok = wt[j] != nullptr;
        for (int k = 0; weights_ok && k < h->prog->A; ++k) {
            weights_ok = ok4(wt[j][k]);
            sa.w[j][k] = wt[j][k];
        }
    }
    int r = rcritic_args(h, h ? h->prog->gru_sep_fn[3] : nullptr, obs_record_n, final_obs_n, n_steps, episode_length,
                         weights_ok, rnn_state, rnn_state_record, values, final_values, net_flags, ln_eps, sa.c);
    if (r) return r;
    NvtxRange range("mpe_critic_gru_separated");
    return launch_rcritic(h, h->prog->gru_sep_fn[3], &sa, static_cast<unsigned>(h->prog->A), h->prog->critic_gru_floats,
                          stream, "cudaLaunchKernelExC(critic_gru_separated)");
}

static int64_t gae_scan_blocks(const mpe_env *h) { return (h->prog->A * h->n + kGaeThreads - 1) / kGaeThreads; }

extern "C" int64_t mpe_gae_workspace_bytes(mpe_handle h) {
    return h ? kGaeWsHeader + 16 * gae_scan_blocks(h) : static_cast<int64_t>(MPE_ERR_BAD_ARG);
}

extern "C" int mpe_gae(mpe_handle h, const float *rewards, const float *values, const float *final_values,
                       int32_t n_steps, int32_t episode_length, float gamma, float gae_lambda, uint32_t flags,
                       const float *value_norm, float *returns, float *advantages, void *workspace,
                       int64_t workspace_bytes, void *stream) {
    if (!h || n_steps < 1) return MPE_ERR_BAD_ARG;
    if (h->device < 0) return MPE_ERR_NO_DEVICE;
    if (episode_length < 0 || (episode_length > 0 && n_steps % episode_length != 0)) return MPE_ERR_BAD_ARG;
    if (!(gamma >= 0.0f && gamma <= 1.0f) || !(gae_lambda >= 0.0f && gae_lambda <= 1.0f)) return MPE_ERR_BAD_ARG;
    if (flags & ~(kGaeBootstrap | kGaeNormalize | kGaePerAgentNorm)) return MPE_ERR_BAD_ARG;
    const bool norm = flags & kGaeNormalize;
    if (!ok4(rewards) || !ok4(values) || !ok4(returns) || !ok4(advantages) ||
        ((flags & kGaeBootstrap) && !ok4(final_values)) || (value_norm != nullptr && !ok4(value_norm)) ||
        ((flags & kGaePerAgentNorm) && value_norm == nullptr) ||
        (norm && (!ok8(workspace) || workspace_bytes < mpe_gae_workspace_bytes(h))))
        return MPE_ERR_BAD_ARG;
    GaeArgs a{};
    a.rew = rewards; a.val = values; a.final_val = (flags & kGaeBootstrap) ? final_values : nullptr;
    a.value_norm = value_norm; a.ret = returns; a.adv = advantages;
    char *ws = static_cast<char *>(workspace);
    if (norm) {
        a.stats = reinterpret_cast<double *>(ws);
        a.ticket = reinterpret_cast<unsigned *>(ws + 16);
        a.partial = reinterpret_cast<double *>(ws + kGaeWsHeader);
    }
    a.cols = h->prog->A * h->n; a.n = h->n;
    a.T = n_steps; a.L = episode_length > 0 ? episode_length : n_steps;
    a.gamma = gamma; a.lambda = gae_lambda; a.flags = flags;
    NvtxRange range("mpe_gae");
    void *params[] = {&a};
    if (norm) {   // the scan's last block is the one that takes ticket blocks - 1
        int prev = 0;
        CUDA_TRY(cudaGetDevice(&prev));
        if (prev != h->device) CUDA_TRY(cudaSetDevice(h->device));
        const cudaError_t e = cudaMemsetAsync(a.ticket, 0, sizeof(unsigned), static_cast<cudaStream_t>(stream));
        if (prev != h->device) cudaSetDevice(prev);
        if (e != cudaSuccess) return cuda_fail(e, "cudaMemsetAsync(gae ticket)");
    }
    int r = launch_kernel(h, gae_kernel(norm ? 1 : 0), gae_scan_blocks(h), kGaeThreads, 0, stream, params, false,
                          "cudaLaunchKernelExC(gae)");
    if (r || !norm) return r;
    const int64_t total = a.cols * n_steps, want = (total + kGaeNormThreads * 4 - 1) / (kGaeNormThreads * 4);
    const int64_t cap = 8 * static_cast<int64_t>(h->sms > 0 ? h->sms : 1);   // 2048 threads per SM, grid-stride
    return launch_kernel(h, gae_kernel(2), want < cap ? want : cap, kGaeNormThreads, 0, stream, params, false,
                         "cudaLaunchKernelExC(gae_normalize)");
}

// adjacent (dst, src, bytes) copies with equal small gaps on both sides are issued as one DMA
struct CopySeg { char *dst; const char *src; size_t bytes; };
static int issue_copies(CopySeg *seg, int n, cudaMemcpyKind kind, cudaStream_t s, const char *what, bool coalesce) {
    int i = 0;
    while (i < n) {
        CopySeg cur = seg[i++];
        while (coalesce && i < n) {
            const ptrdiff_t gd = seg[i].dst - (cur.dst + cur.bytes), gs = seg[i].src - (cur.src + cur.bytes);
            if (gd != gs || gd < 0 || gd >= 512) break;
            cur.bytes += static_cast<size_t>(gd) + seg[i].bytes;
            ++i;
        }
        cudaError_t e = cudaMemcpyAsync(cur.dst, cur.src, cur.bytes, kind, s);
        if (e != cudaSuccess) return cuda_fail(e, what);
    }
    return MPE_OK;
}

static int step_range(mpe_handle h, void *pv, const void *lm, float *comm, const int32_t *goal,
                      const float *const *act_n, float *const *obs_n, float *rew, uint8_t *done, float *info,
                      uint32_t flags, void *stream, int64_t begin, int64_t count) {
    if (h->prog->scenario == MPE_SCN_CUSTOM) return MPE_ERR_UNSUPPORTED;
    StepArgs a{};
    int r = fill_state(h, a, pv, lm, comm, goal);
    if (r) return r;
    r = fill_actions(h, a, act_n);
    if (r) return r;
    r = fill_outputs(h, a, obs_n, rew, done, info);
    if (r) return r;
    a.flags = flags;
    return launch(h, kFusedStep, a, stream, begin, count);
}

// floats (4-byte words) per world in act_n[i]: the action vector, or one index per sub-action (discrete_action_input)
static size_t act_row_words(const mpe_env *h, int i, uint32_t flags) {
    if (flags & MPE_FLAG_DISCRETE_ACTION_INPUT) return (h->desc.agent_movable[i] ? 1 : 0) + (h->desc.agent_silent[i] ? 0 : 1);
    return static_cast<size_t>(h->prog->act_dim[i]);
}

static int64_t host_chunk_min() {  // MPE_B200_HOST_CHUNK_MIN: smallest batch that is pipelined (default 262144)
    static const int64_t m = [] { const char *e = getenv("MPE_B200_HOST_CHUNK_MIN"); return e ? atoll(e) : 262144LL; }();
    return m;
}
static int host_chunks() {  // MPE_B200_HOST_CHUNKS: 1 disables the pipeline (default 4)
    static const int c = [] { const char *e = getenv("MPE_B200_HOST_CHUNKS"); int v = e ? atoi(e) : 4; return v < 1 ? 1 : (v > 16 ? 16 : v); }();
    return c;
}

extern "C" int mpe_step_host(mpe_handle h, void *pv, const void *lm, float *comm, const int32_t *goal,
                             const float *const *act_n_host, float *const *act_n_dev, float *const *obs_n_dev,
                             float *rew_dev, uint8_t *done_dev, float *info_dev, float *const *obs_n_host,
                             float *rew_host, uint8_t *done_host, float *info_host, uint32_t flags, void *stream) {
    if (!h || !act_n_host || !act_n_dev || !obs_n_host || !obs_n_dev || !rew_host || !done_host) return MPE_ERR_BAD_ARG;
    if (h->device < 0) return MPE_ERR_NO_DEVICE;
    NvtxRange range("mpe_step_host");
    const Program *p = h->prog;
    cudaStream_t user = static_cast<cudaStream_t>(stream);
    const size_t n = static_cast<size_t>(h->n);
    for (int i = 0; i < p->A; ++i)
        if (!act_n_host[i] || !act_n_dev[i] || !obs_n_host[i] || !obs_n_dev[i]) return MPE_ERR_BAD_ARG;
    const bool want_info = info_host && info_dev && p->INFO > 0;
    int prev = 0;
    CUDA_TRY(cudaGetDevice(&prev));
    if (prev != h->device) CUDA_TRY(cudaSetDevice(h->device));
    int rc = MPE_OK;
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    cudaStreamIsCapturing(user, &cap);
    // below ~256k worlds the extra copy calls cost more than the overlap gains
    const int chunks = (h->n >= host_chunk_min() && cap == cudaStreamCaptureStatusNone) ? host_chunks() : 1;
    if (chunks == 1) {
        // small batches: one H2D per agent, one launch, one coalesced D2H
        CopySeg seg[kMaxA + 3];
        int ns = 0;
        for (int i = 0; i < p->A; ++i)
            seg[ns++] = {reinterpret_cast<char *>(act_n_dev[i]), reinterpret_cast<const char *>(act_n_host[i]),
                         sizeof(float) * n * act_row_words(h, i, flags)};
        rc = issue_copies(seg, ns, cudaMemcpyHostToDevice, user, "cudaMemcpyAsync(H2D actions)", false);
        if (rc == MPE_OK)
            rc = step_range(h, pv, lm, comm, goal, act_n_dev, obs_n_dev, rew_dev, done_dev, want_info ? info_dev : nullptr,
                            flags, stream, 0, h->n);
        if (rc == MPE_OK) {
            ns = 0;
            for (int i = 0; i < p->A; ++i)
                seg[ns++] = {reinterpret_cast<char *>(obs_n_host[i]), reinterpret_cast<const char *>(obs_n_dev[i]),
                             sizeof(float) * n * p->obs_dim[i]};
            seg[ns++] = {reinterpret_cast<char *>(rew_host), reinterpret_cast<const char *>(rew_dev), sizeof(float) * n * p->A};
            seg[ns++] = {reinterpret_cast<char *>(done_host), reinterpret_cast<const char *>(done_dev), n * p->A};
            if (want_info)
                seg[ns++] = {reinterpret_cast<char *>(info_host), reinterpret_cast<const char *>(info_dev),
                             sizeof(float) * n * p->A * p->INFO};
            rc = issue_copies(seg, ns, cudaMemcpyDeviceToHost, user, "cudaMemcpyAsync(D2H obs/rew/done/info)",
                              (flags & MPE_FLAG_HOST_SLAB) != 0);
        }
    } else {
        // Large batches: the worlds are cut into `chunks` ranges (multiples of 128 worlds, so every tile stays
        // 16-byte aligned) that alternate between two internal streams: while chunk c drains over the D2H copy
        // engine, chunk c+1 uploads its actions and computes.  The caller's stream forks into and joins the two.
        cudaError_t e = cudaEventRecord(h->ev_fork, user);
        for (int k = 0; k < 2 && e == cudaSuccess; ++k) e = cudaStreamWaitEvent(h->aux[k], h->ev_fork, 0);
        if (e != cudaSuccess) rc = cuda_fail(e, "mpe_step_host: fork");
        const int64_t per = ((h->n + chunks - 1) / chunks + 127) / 128 * 128;
        for (int c = 0; c < chunks && rc == MPE_OK; ++c) {
            const int64_t begin = c * per;
            if (begin >= h->n) break;
            const int64_t count = (begin + per <= h->n) ? per : h->n - begin;
            cudaStream_t s = h->aux[c & 1];
            for (int i = 0; i < p->A && e == cudaSuccess; ++i)
                e = cudaMemcpyAsync(act_n_dev[i] + begin * act_row_words(h, i, flags), act_n_host[i] + begin * act_row_words(h, i, flags),
                                    sizeof(float) * count * act_row_words(h, i, flags), cudaMemcpyHostToDevice, s);
            if (e != cudaSuccess) { rc = cuda_fail(e, "cudaMemcpyAsync(H2D actions)"); break; }
            rc = step_range(h, pv, lm, comm, goal, act_n_dev, obs_n_dev, rew_dev, done_dev, want_info ? info_dev : nullptr,
                            flags, s, begin, count);
            if (rc != MPE_OK) break;
            for (int i = 0; i < p->A && e == cudaSuccess; ++i)
                e = cudaMemcpyAsync(obs_n_host[i] + begin * p->obs_dim[i], obs_n_dev[i] + begin * p->obs_dim[i],
                                    sizeof(float) * count * p->obs_dim[i], cudaMemcpyDeviceToHost, s);
            if (e == cudaSuccess)   // rew / done / info are [rows][n_env]: one strided copy per array
                e = cudaMemcpy2DAsync(rew_host + begin, sizeof(float) * n, rew_dev + begin, sizeof(float) * n,
                                      sizeof(float) * count, p->A, cudaMemcpyDeviceToHost, s);
            if (e == cudaSuccess)
                e = cudaMemcpy2DAsync(done_host + begin, n, done_dev + begin, n, count, p->A, cudaMemcpyDeviceToHost, s);
            if (e == cudaSuccess && want_info)
                e = cudaMemcpy2DAsync(info_host + begin, sizeof(float) * n, info_dev + begin, sizeof(float) * n,
                                      sizeof(float) * count, static_cast<size_t>(p->A) * p->INFO, cudaMemcpyDeviceToHost, s);
            if (e != cudaSuccess) rc = cuda_fail(e, "cudaMemcpyAsync(D2H chunk)");
        }
        for (int k = 0; k < 2; ++k) {   // join, even after an error, so that the caller's stream stays ordered
            cudaError_t j = cudaEventRecord(h->ev_join[k], h->aux[k]);
            if (j == cudaSuccess) j = cudaStreamWaitEvent(user, h->ev_join[k], 0);
            if (j != cudaSuccess && rc == MPE_OK) rc = cuda_fail(j, "mpe_step_host: join");
        }
    }
    if (prev != h->device) cudaSetDevice(prev);
    return rc;
}

static int reset_impl(mpe_handle h, void *pv, void *lm, float *comm, int32_t *goal, const uint8_t *mask,
                      uint64_t seed, uint64_t world_offset, uint64_t epoch, unsigned long long *epoch_dev, void *stream) {
    if (!h) return MPE_ERR_BAD_ARG;
    if (h->device < 0) return MPE_ERR_NO_DEVICE;
    NvtxRange range("mpe_reset");
    StepArgs tmp{};
    int r = fill_state(h, tmp, pv, lm, comm, goal);
    if (r) return r;
    const Program *p = h->prog;
    ResetArgs a{};
    a.n = h->n; a.A = p->A; a.L = p->L; a.NC = p->NS * p->DIMC; a.G = p->G;
    a.pv = static_cast<float4 *>(pv); a.lm = static_cast<float2 *>(lm); a.comm = comm; a.goal = goal; a.mask = mask;
    a.seed = seed; a.world_offset = world_offset; a.epoch = epoch; a.epoch_dev = epoch_dev;
    a.landmark_range = reset_landmark_range(p->scenario);
    a.goal_mod = p->L > 0 ? p->L : 1;
    void *params[] = {&a};
    r = launch_kernel(h, reinterpret_cast<const void *>(reset_kernel), (h->n + 255) / 256, 256, 0, stream, params, false,
                      "reset_kernel");
    if (r == MPE_OK && epoch_dev) {   // the device epoch advances after this reset has read it
        void *bump[] = {&epoch_dev};
        r = launch_kernel(h, reinterpret_cast<const void *>(bump_epoch_kernel), 1, 1, 0, stream, bump, false, "reset_kernel");
    }
    return r;
}

extern "C" int mpe_reset(mpe_handle h, void *pv, void *lm, float *comm, int32_t *goal, const uint8_t *mask,
                         uint64_t seed, uint64_t world_offset, uint64_t epoch, void *stream) {
    return reset_impl(h, pv, lm, comm, goal, mask, seed, world_offset, epoch, nullptr, stream);
}

extern "C" int mpe_reset_dev_epoch(mpe_handle h, void *pv, void *lm, float *comm, int32_t *goal, const uint8_t *mask,
                                   uint64_t seed, uint64_t world_offset, unsigned long long *epoch_dev, void *stream) {
    if (!epoch_dev) return MPE_ERR_BAD_ARG;
    return reset_impl(h, pv, lm, comm, goal, mask, seed, world_offset, 0, epoch_dev, stream);
}

extern "C" int mpe_probe_stream(int device, const void *src, int64_t read_bytes, void *dst, int64_t write_bytes,
                                int64_t threads, void *stream) {
    if (!ok16(src) || !ok16(dst) || read_bytes < 0 || write_bytes < 0 || threads < 256) return MPE_ERR_BAD_ARG;
    int prev = 0;
    CUDA_TRY(cudaGetDevice(&prev));
    if (prev != device) CUDA_TRY(cudaSetDevice(device));
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(static_cast<unsigned>((threads + 255) / 256));
    cfg.blockDim = dim3(256);
    cfg.stream = static_cast<cudaStream_t>(stream);
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_mode() ? 1 : 0;
    const float4 *s4 = static_cast<const float4 *>(src);
    float4 *d4 = static_cast<float4 *>(dst);
    long long nr = read_bytes / 16, nw = write_bytes / 16;
    void *params[] = {&s4, &nr, &d4, &nw};
    cudaError_t e = cudaLaunchKernelExC(&cfg, reinterpret_cast<const void *>(stream_probe_kernel), params);
    if (prev != device) cudaSetDevice(prev);
    if (e != cudaSuccess) return cuda_fail(e, "cudaLaunchKernelExC(stream_probe)");
    return MPE_OK;
}

extern "C" const char *mpe_strerror(int err) {
    switch (err) {
    case MPE_OK: return "ok";
    case MPE_ERR_BAD_ARG: return "bad argument (null or misaligned pointer, bad size or index)";
    case MPE_ERR_BAD_DESC: return "descriptor does not fit its scenario program";
    case MPE_ERR_UNSUPPORTED: return "no compiled sm_90a program for this scenario / shape / flag";
    case MPE_ERR_CUDA: return "CUDA runtime error (see mpe_last_cuda_error)";
    case MPE_ERR_NO_DEVICE: return "no sm_90 (H100) device with that index, or shape-only handle (device -1)";
    default: return "unknown error";
    }
}
extern "C" const char *mpe_last_cuda_error(void) { return g_cuda_err; }
extern "C" int mpe_abi_version(void) { return MPE_ABI_VERSION; }
extern "C" int64_t mpe_kernel_launches(void) { return __atomic_load_n(&g_launches, __ATOMIC_RELAXED); }
#endif  // MPE_KERNEL_TEMPLATES_ONLY
