/*
 * mpe_b200.h -- C ABI of libmpe_b200.so: batched multi-agent particle worlds on H100 (sm_90a).
 *
 * The reference (openai/multiagent-particle-envs) exposes a *Python* API and no FFI; each entry
 * point below names the reference interface (file:line under /root/reference) whose work it
 * replaces for a batch of n_env independent worlds.  See INTEGRATION.md for the ctypes binding a
 * maintainer of the reference would add.
 *
 * Conventions
 *   - plain pointers and sizes only; no C++/torch types cross this boundary;
 *   - every pointer marked "dev" is a device pointer on the handle's device, borrowed for the
 *     duration of the stream-ordered call; the library allocates nothing per step;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream);
 *   - every function returns 0 on success or a negative MPE_ERR_* code; mpe_strerror() names it;
 *   - calls are asynchronous w.r.t. the host; a handle is bound to one device and is not
 *     thread-safe (the reference is single-threaded too: environment.py:80-104).
 *
 * Device state layout (fp32, struct-of-arrays over the world index w in [0, n_env)):
 *   agent_pv  float4 [A][n_env]        (p_pos.x, p_pos.y, p_vel.x, p_vel.y)   core.py:4-9
 *   lm_p      float2 [L][n_env]        landmark p_pos (landmarks never move in any scenario)
 *   comm      float  [S*dim_c][n_env]  state.c of the S non-silent agents     core.py:11-16
 *   goal      int32  [G][n_env]        per-world goal indices (push/adversary/... scenarios)
 * API-facing per-agent tensors are row-major exactly as a trainer holds them:
 *   act_n[i]  float  [n_env][act_dim_i]  (5 physical one-hot/probabilities, then dim_c comm)
 *   obs_n[i]  float  [n_env][obs_dim_i]    (base pointer 16-byte aligned; act_n[i] may be 4-byte aligned,
 *                                           16-byte alignment enables the cp.async path)
 *   rew       float  [A][n_env],  done uint8 [A][n_env],  info float [A][info_dim][n_env]
 */
#ifndef MPE_B200_H
#define MPE_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define MPE_API __attribute__((visibility("default")))
#else
#define MPE_API
#endif

#define MPE_ABI_VERSION 1
#define MPE_MAX_AGENTS 8
#define MPE_MAX_LANDMARKS 8

/* scenario programs (multiagent/scenarios/<name>.py) */
enum mpe_scenario {
    MPE_SCN_SIMPLE = 0,           /* simple.py */
    MPE_SCN_SPREAD = 1,           /* simple_spread.py (A = L = N) */
    MPE_SCN_TAG = 2,              /* simple_tag.py */
    MPE_SCN_WORLD_COMM = 3,       /* simple_world_comm.py */
    MPE_SCN_ADVERSARY = 4,        /* simple_adversary.py */
    MPE_SCN_PUSH = 5,             /* simple_push.py */
    MPE_SCN_SPEAKER_LISTENER = 6, /* simple_speaker_listener.py */
    MPE_SCN_REFERENCE = 7,        /* simple_reference.py */
    MPE_SCN_CRYPTO = 8,           /* simple_crypto.py */
    MPE_SCN_CUSTOM = 9,           /* user scenario: native _set_action + World.step for ANY entity table (<= 8 agents,
                                     <= 8 landmarks); observation / reward stay in the caller's (GPU) code, so only
                                     mpe_set_action, mpe_world_step and mpe_reset are available */
    MPE_SCN_COUNT_
};

/* error codes */
enum mpe_error {
    MPE_OK = 0,
    MPE_ERR_BAD_ARG = -1,         /* null/misaligned pointer, n_env <= 0, bad agent index */
    MPE_ERR_BAD_DESC = -2,        /* descriptor inconsistent with its scenario program */
    MPE_ERR_UNSUPPORTED = -3,     /* no compiled kernel for this scenario/shape */
    MPE_ERR_CUDA = -4,            /* CUDA runtime error; see mpe_last_cuda_error() */
    MPE_ERR_NO_DEVICE = -5        /* no sm_90 device / device index out of range */
};

/* step flags (MultiAgentEnv attributes, environment.py:29-35) */
enum mpe_step_flags {
    MPE_FLAG_SHARED_REWARD = 1,         /* env.shared_reward: every agent gets sum_i r_i   :100-102 */
    MPE_FLAG_FORCE_DISCRETE_ACTION = 2, /* env.force_discrete_action: argmax one-hot       :169-172 */
    MPE_FLAG_DISCRETE_ACTION_INPUT = 4, /* env.discrete_action_input (:161-167,185-187): act_n[i] is int32
                                           [n_env][n_sub_i], one index per sub-action -- movement (0 none, 1 -x,
                                           2 +x, 3 -y, 4 +y) if the agent is movable, then the utterance
                                           (one-hot of the index) if it is not silent; decoded inside the kernel */
    MPE_FLAG_HOST_SLAB = 8              /* mpe_step_host only: obs_n_host[0..A), rew_host, done_host (, info_host)
                                           are consecutive parts of ONE host allocation and their device
                                           counterparts of ONE device allocation, with equal gaps < 512 B:
                                           the D2H copies are coalesced into a single DMA */
};

/*
 * Immutable world descriptor: what Scenario.make_world() writes onto World / Entity objects
 * (core.py:25-99 defaults; e.g. simple_spread.py:7-29), flattened.  Doubles keep the Python
 * values exact; the library rounds derived constants to fp32 once at create time.
 */
typedef struct mpe_desc {
    int32_t abi_version;                       /* MPE_ABI_VERSION */
    int32_t scenario;                          /* enum mpe_scenario */
    int32_t n_agents;                          /* len(world.agents) == len(world.policy_agents) */
    int32_t n_landmarks;                       /* len(world.landmarks) */
    int32_t dim_c;                             /* world.dim_c                       core.py:88 */
    int32_t n_adversaries;                     /* agents [0, n_adv) have .adversary (tag/world_comm/adversary/push) */
    int32_t n_obstacles;                       /* world_comm: landmarks = obstacles ++ food ++ forests */
    int32_t n_food;
    int32_t n_forests;
    int32_t reserved_i[7];
    double dt;                                 /* core.py:94  */
    double damping;                            /* core.py:96  */
    double contact_force;                      /* core.py:98  */
    double contact_margin;                     /* core.py:99  */
    double agent_size[MPE_MAX_AGENTS];         /* core.py:32  */
    double agent_mass[MPE_MAX_AGENTS];         /* core.py:47-51 */
    double agent_sens[MPE_MAX_AGENTS];         /* accel or 5.0: environment.py:178-181 */
    double agent_max_speed[MPE_MAX_AGENTS];    /* < 0 means None: core.py:41,164 */
    double landmark_size[MPE_MAX_LANDMARKS];
    uint8_t agent_movable[MPE_MAX_AGENTS];     /* core.py:58  */
    uint8_t agent_collide[MPE_MAX_AGENTS];     /* core.py:36  */
    uint8_t agent_silent[MPE_MAX_AGENTS];      /* core.py:60  */
    uint8_t agent_adversary[MPE_MAX_AGENTS];
    uint8_t agent_leader[MPE_MAX_AGENTS];      /* simple_world_comm.py:23 */
    uint8_t landmark_collide[MPE_MAX_LANDMARKS];
    uint8_t reserved_b[16];
} mpe_desc;

typedef struct mpe_env *mpe_handle;

/* ---- lifetime -------------------------------------------------------------------------- */

/* Validates the descriptor against its scenario program and binds a batch of n_env worlds to a
 * device.  Replaces: World() + Scenario.make_world() + MultiAgentEnv.__init__ shape discovery
 * (make_env.py:36-43, environment.py:14-78). */
MPE_API int mpe_create(const mpe_desc *desc, int64_t n_env, int device, mpe_handle *out);
MPE_API int mpe_destroy(mpe_handle h);

/* ---- shape queries (environment.py:39-70: action_space / observation_space construction) -- */
MPE_API int mpe_num_agents(mpe_handle h);
MPE_API int64_t mpe_num_envs(mpe_handle h);
MPE_API int mpe_obs_dim(mpe_handle h, int agent);     /* len(scenario.observation(agent, world)) :68 */
MPE_API int mpe_act_dim(mpe_handle h, int agent);     /* 5 if movable (+ dim_c if not silent)    :45-63 */
MPE_API int mpe_num_speakers(mpe_handle h);           /* S: agents with silent == False */
MPE_API int mpe_num_goals(mpe_handle h);              /* G: rows of the goal tensor */
MPE_API int mpe_info_dim(mpe_handle h);               /* floats of benchmark_data per agent */
MPE_API int64_t mpe_bytes_per_env_step(mpe_handle h); /* compulsory HBM bytes of one fused step (SURVEY 8d) */

/* ---- reset (scenario.reset_world: e.g. simple_spread.py:31-45; environment.py:106-116) ---- */
/* Worlds with mask[w] != 0 (all if mask == NULL) get i.i.d. uniform positions from a Philox4x32
 * stream keyed by (seed, world_offset + w, epoch): results do not depend on how the batch is
 * sharded.  Velocities, comm state are zeroed; goal indices redrawn. */
MPE_API int mpe_reset(mpe_handle h, void *agent_pv_dev, void *lm_p_dev, float *comm_dev, int32_t *goal_dev,
              const uint8_t *mask_dev, uint64_t seed, uint64_t world_offset, uint64_t epoch,
              void *stream);

/* Same reset, but the epoch is read from device memory (*epoch_dev) and incremented afterwards on the stream:
 * a reset captured in a CUDA graph then draws fresh initial conditions on every replay. */
MPE_API int mpe_reset_dev_epoch(mpe_handle h, void *agent_pv_dev, void *lm_p_dev, float *comm_dev, int32_t *goal_dev,
                                const uint8_t *mask_dev, uint64_t seed, uint64_t world_offset,
                                unsigned long long *epoch_dev, void *stream);

/* ---- the hot path ------------------------------------------------------------------------ */

/* MultiAgentEnv._set_action for all agents (environment.py:144-192): act_n -> action.u, action.c.
 * u: float2 [A][n_env]; c: float [S*dim_c][n_env]. */
MPE_API int mpe_set_action(mpe_handle h, const float *const *act_n_dev, float *u_dev, float *c_dev,
                   uint32_t flags, void *stream);

/* World.step (core.py:117-131): apply_action_force, apply_environment_force /
 * get_collision_force, integrate_state, update_agent_state -- from already decoded actions. */
MPE_API int mpe_world_step(mpe_handle h, void *agent_pv_dev, const void *lm_p_dev, float *comm_dev,
                   const float *u_dev, const float *c_dev, void *stream);

/* scenario.observation / reward / benchmark_data for every agent plus the done/shared-reward
 * glue of MultiAgentEnv.step (environment.py:92-102,119-141) on the current state.
 * info_dev may be NULL. */
MPE_API int mpe_observe(mpe_handle h, const void *agent_pv_dev, const void *lm_p_dev, const float *comm_dev,
                const int32_t *goal_dev, float *const *obs_n_dev, float *rew_dev, uint8_t *done_dev,
                float *info_dev, uint32_t flags, void *stream);

/* MultiAgentEnv.step (environment.py:80-104) fused into one launch:
 * _set_action -> World.step -> observation/reward/done/info -> shared-reward sum. */
MPE_API int mpe_step(mpe_handle h, void *agent_pv_dev, const void *lm_p_dev, float *comm_dev,
             const int32_t *goal_dev, const float *const *act_n_dev, float *const *obs_n_dev,
             float *rew_dev, uint8_t *done_dev, float *info_dev, uint32_t flags, void *stream);

/* n_steps consecutive MultiAgentEnv.step calls (environment.py:80-104; the loop of bin/interactive.py:27-39 with the
 * policy's outputs known in advance) on pre-generated actions, in ONE launch: act_seq_dev[i] is float
 * [n_steps][n_env][act_dim_i].  A world's state stays in registers between the steps; per step only the actions are read.
 * Outputs: the state after the last step, obs_n_dev / done_dev for that final state, rew_sum_dev [A][n_env] = the
 * per-agent rewards summed over the steps in step order, and -- if rew_steps_dev is not NULL -- every step's rewards
 * [n_steps][A][n_env].  Bit-identical to n_steps calls of mpe_step.  (CEM / MPPI style planners, evaluation of
 * recorded action sequences.)  MPE_FLAG_DISCRETE_ACTION_INPUT is not supported here. */
MPE_API int mpe_rollout(mpe_handle h, void *agent_pv_dev, const void *lm_p_dev, float *comm_dev,
                        const int32_t *goal_dev, const float *const *act_seq_dev, int32_t n_steps,
                        float *const *obs_n_dev, float *rew_sum_dev, float *rew_steps_dev, uint8_t *done_dev,
                        uint32_t flags, void *stream);

/* n_steps consecutive MultiAgentEnv.step calls in ONE launch with the policy INSIDE the kernel (the trainer's loop
 * obs -> actor network -> env.step, bin/interactive.py:27-39 with `policy.action(obs_n[i])` being a small actor): agent i
 * acts with  a_i = softmax(W2_i . relu(W1_i^T . obs_i + b1_i) + b2_i),  obs_dim_i -> hidden -> 5 movement probabilities.
 * w1_n[i]: float [obs_dim_i][hidden] (input-major, 16-byte aligned), b1_n[i]: [hidden], w2_n[i]: [5][hidden], b2_n[i]: [5];
 * hidden = 32 or 64.  World state stays in registers, observations are never written between steps.  Outputs as
 * mpe_rollout; act_record_n (NULL or per agent float [n_steps][n_env][5]) receives the actions taken -- feeding them to
 * mpe_rollout / mpe_step reproduces state, observations and reward sums bit for bit.  Only for scenarios whose agents
 * all move and are silent and for which the program was built (the BASELINE.json worlds simple, simple_spread N = 3,
 * simple_tag 3 + 1); otherwise MPE_ERR_UNSUPPORTED. */
MPE_API int mpe_rollout_policy(mpe_handle h, void *agent_pv_dev, const void *lm_p_dev, float *comm_dev,
                               const int32_t *goal_dev, const float *const *w1_n, const float *const *b1_n,
                               const float *const *w2_n, const float *const *b2_n, int32_t hidden, int32_t n_steps,
                               float *const *obs_n_dev, float *rew_sum_dev, float *rew_steps_dev,
                               float *const *act_record_n, uint8_t *done_dev, uint32_t flags, void *stream);

/* The same closed-loop rollout with MADDPG's actor (mlp_model): obs_dim_i -> hidden -> ReLU -> hidden -> ReLU -> act_dim_i,
 *     logits_i = W3_i relu(W2_i relu(W1_i obs_i + b1_i) + b2_i) + b3_i,
 * evaluated on the tensor cores (TF32 mma.sync, fp32 accumulation; every operand -- observations, both hidden layers and
 * all weights -- rounded to TF32 with round-to-nearest, ties away from zero; biases added in fp32).  Weights in torch
 * nn.Linear layout: w1_n[i] float [hidden][obs_dim_i], b1_n[i] [hidden], w2_n[i] [hidden][hidden], b2_n[i] [hidden],
 * w3_n[i] [act_dim_i][hidden], b3_n[i] [act_dim_i]; hidden = 32 or 64 (both hidden layers).
 * The act_dim_i logits split into the action vector's sub-spaces (environment.py:40-66): 5 movement logits if agent i
 * is movable, then dim_c utterance logits if it is not silent.  explore == 0: the action is the concatenation of one
 * softmax per sub-space (MADDPG's mode()).  explore != 0: of one Gumbel-softmax sample softmax(z - log(-log u)) per
 * sub-space (SoftCategoricalPd / SoftMultiCategoricalPd.sample).  Logit k uses u_k = word k mod 4 of the Philox4x32-10
 * block b = k div 4 with key = explore_seed and counter = (world_offset + w lo, hi, explore_epoch lo,
 * 0x40000000 | ((t * A + i) * S + b)), S = 2 when every act_dim of the scenario is <= 8 and 4 otherwise
 * (simple_reference); u = ((bits >> 8) + 0.5) * 2^-24 with the sum rounded toward zero in fp32.  The draw depends on the
 * global world index, not on the batch it runs in.  An exploring call with n_steps * A * S > 2^30 is refused with
 * MPE_ERR_BAD_ARG before anything runs.
 * The action is applied as _set_action does: movement (p1 - p2, p3 - p4) * sensitivity for movable agents only (an
 * immovable agent's state is never written), the utterance becomes action.c; after the physics state.c = action.c and
 * the rewards are computed from the new state, so an utterance of step t reaches the observations from step t + 1 on.
 * comm_dev is read at the start and written at the end.
 * Records (NULL: not written): act_record_n[i] float [n_steps][n_env][act_dim_i], the action applied (the sample when
 * exploring); obs_record_n[i] float [n_steps][n_env][obs_dim_i] (16-byte aligned), the observation agent i acted on at
 * step t; rew_steps_dev as in mpe_rollout_policy.  Feeding act_record_n to mpe_step reproduces state, comm state,
 * observations and rewards bit for bit.  Built for simple, simple_spread N = 2 to 6, simple_tag 3 + 1, 1 + 1, 2 + 1,
 * 4 + 2 and 6 + 2 (3 landmarks), simple_speaker_listener, simple_reference, simple_crypto, simple_adversary (1 + 2 and
 * 1 + 3 agents) and simple_push (1 + 1); otherwise (simple_world_comm), or for another hidden width,
 * MPE_ERR_UNSUPPORTED.  The scenario and hidden width are checked before any
 * state, weight or output pointer: a call with those null returns MPE_ERR_UNSUPPORTED or MPE_ERR_BAD_ARG and runs
 * nothing. */
MPE_API int mpe_rollout_policy_mlp(mpe_handle h, void *agent_pv_dev, const void *lm_p_dev, float *comm_dev,
                                   const int32_t *goal_dev, const float *const *w1_n, const float *const *b1_n,
                                   const float *const *w2_n, const float *const *b2_n, const float *const *w3_n,
                                   const float *const *b3_n, int32_t hidden, int32_t n_steps, int32_t explore,
                                   uint64_t explore_seed, uint64_t explore_epoch, uint64_t world_offset,
                                   float *const *obs_n_dev, float *rew_sum_dev, float *rew_steps_dev,
                                   float *const *act_record_n, float *const *obs_record_n, uint8_t *done_dev,
                                   uint32_t flags, void *stream);

/* n_episodes MADDPG episodes of episode_length steps each in ONE launch: mpe_rollout_policy_mlp with the reset between
 * episodes inside the kernel.  Bit for bit the same as, for e = 0 .. n_episodes - 1, mpe_rollout_policy_mlp(n_steps =
 * episode_length, explore_epoch + e) followed by mpe_reset(reset_seed, world_offset, reset_epoch + e) without a mask:
 *  - exploration: episode e uses explore epoch explore_epoch + e and its step counter t restarts at 0, so an exploring
 *    call with episode_length * A * S > 2^30 is refused with MPE_ERR_BAD_ARG before anything runs;
 *  - reset: after the last step of episode e every world is redrawn as mpe_reset draws it with epoch reset_epoch + e
 *    (agents, immovable ones included, at U(-1, 1)^2 and at rest, landmarks, comm 0, goals), so lm_p_dev and goal_dev are
 *    written;
 *  - records span all n_episodes * episode_length steps, at global step e * episode_length + t: rew_steps_dev
 *    [T][A][n_env], act_record_n[i] [T][n_env][act_dim_i], obs_record_n[i] [T][n_env][obs_dim_i];
 *  - final_obs_record_n (NULL, or one 16-byte aligned pointer for every agent): [n_episodes][n_env][obs_dim_i], the
 *    observation after the last step of episode e, before its reset (MADDPG's new_obs of the terminal transition);
 *  - ep_rew_dev [n_episodes][A][n_env]: each episode's per-agent rewards summed in step order;
 *  - obs_n_dev: the observations of the state after the last reset; done_dev: all 0.
 * The state arrays end as the last reset left them.  episode_length and n_episodes must be >= 1 with a product below
 * 2^31 (else MPE_ERR_BAD_ARG).  Built for the programs of mpe_rollout_policy_mlp; the scenario and hidden width are
 * checked before any pointer, as there. */
MPE_API int mpe_rollout_policy_mlp_episodes(mpe_handle h, void *agent_pv_dev, void *lm_p_dev, float *comm_dev,
                                            int32_t *goal_dev, const float *const *w1_n, const float *const *b1_n,
                                            const float *const *w2_n, const float *const *b2_n, const float *const *w3_n,
                                            const float *const *b3_n, int32_t hidden, int32_t episode_length,
                                            int32_t n_episodes, int32_t explore, uint64_t explore_seed,
                                            uint64_t explore_epoch, uint64_t reset_seed, uint64_t reset_epoch,
                                            uint64_t world_offset, float *const *obs_n_dev, float *ep_rew_dev,
                                            float *rew_steps_dev, float *const *act_record_n, float *const *obs_record_n,
                                            float *const *final_obs_record_n, uint8_t *done_dev, uint32_t flags,
                                            void *stream);

/* Policy-gradient (PPO / A2C) experience with the same actor: mpe_rollout_policy_mlp and mpe_rollout_policy_mlp_episodes
 * with categorical actions.  The logits z are those of the default form (same TF32 GEMMs); then, per action sub-space in
 * action-vector order (5 movement logits if movable, then dim_c utterance logits if not silent):
 *  - explore != 0: k = argmax_c (z_c - log(-log u_c)) with the u of the default form's exploration (same Philox counters,
 *    stride S, epochs, episode step restart), so k is the arg-max of the Gumbel-softmax sample that form would take;
 *    explore == 0: k = argmax_c z_c.  Ties go to the lowest index.
 *  - the action applied is the one-hot vector of k, concatenated over sub-spaces, through the same _set_action arithmetic
 *    as any float action vector: bit for bit what mpe_step does with that one-hot vector.  A speaker's utterance becomes
 *    a one-hot comm state after the physics.
 *  - its log-probability is the sum over sub-spaces, in order, of (z_k - m) - logf(sum_c expf(z_c - m)), m the maximum
 *    of the unperturbed segment, the sum in index order with round-to-nearest adds: Categorical(logits=z).log_prob(k) on
 *    the logits the kernel acted with.
 * k is the POSITION IN THE LOGIT SEGMENT (the one-hot convention, environment.py:173-175), NOT the discrete_action_input
 * code (environment.py:164-167): movement index 1 is +x here, -x there.  Replay the indices as one-hot float vectors.
 * Records (NULL: not written): act_index_record_n[i] int32 [n_steps][n_env][n_sub_i] (n_sub_i = 1 or 2 sub-spaces,
 * movement first), logp_steps_dev float [n_steps][A][n_env] (the layout of rew_steps_dev); everything else, the refusals
 * (scenario and hidden width before any pointer, the exploration counter limit) and the programs built are those of the
 * default form. */
MPE_API int mpe_rollout_policy_mlp_categorical(mpe_handle h, void *agent_pv_dev, const void *lm_p_dev, float *comm_dev,
                                               const int32_t *goal_dev, const float *const *w1_n,
                                               const float *const *b1_n, const float *const *w2_n,
                                               const float *const *b2_n, const float *const *w3_n,
                                               const float *const *b3_n, int32_t hidden, int32_t n_steps, int32_t explore,
                                               uint64_t explore_seed, uint64_t explore_epoch, uint64_t world_offset,
                                               float *const *obs_n_dev, float *rew_sum_dev, float *rew_steps_dev,
                                               float *logp_steps_dev, int32_t *const *act_index_record_n,
                                               float *const *obs_record_n, uint8_t *done_dev, uint32_t flags,
                                               void *stream);
MPE_API int mpe_rollout_policy_mlp_categorical_episodes(
    mpe_handle h, void *agent_pv_dev, void *lm_p_dev, float *comm_dev, int32_t *goal_dev, const float *const *w1_n,
    const float *const *b1_n, const float *const *w2_n, const float *const *b2_n, const float *const *w3_n,
    const float *const *b3_n, int32_t hidden, int32_t episode_length, int32_t n_episodes, int32_t explore,
    uint64_t explore_seed, uint64_t explore_epoch, uint64_t reset_seed, uint64_t reset_epoch, uint64_t world_offset,
    float *const *obs_n_dev, float *ep_rew_dev, float *rew_steps_dev, float *logp_steps_dev,
    int32_t *const *act_index_record_n, float *const *obs_record_n, float *const *final_obs_record_n, uint8_t *done_dev,
    uint32_t flags, void *stream);

/* MAPPO's MLP actor (MLPBase with layer_N = 1 and a categorical ACTLayer head), hidden width 64 only:
 *     [LN(obs_dim_i)] -> Linear(obs_dim_i, 64) -> act -> LN(64) -> Linear(64, 64) -> act -> LN(64) -> Linear(64, act_dim_i)
 * with act = ReLU, or tanh (tanhf) if net_flags & 2; the input LayerNorm only if net_flags & 1.  Every LayerNorm uses
 * ln_eps.  w1_n .. b3_n are the FOLDED network: each LayerNorm's affine (gamma, beta) moved into the Linear after it,
 *     W' = W diag(gamma),   b' = b + W beta
 * (LN(obs) into W1, b1; the first hidden LN into W2, b2; the second into W3, b3), so the kernel normalises without
 * parameters: (x - mu) * rsqrt(var + ln_eps), mu and var two-pass fp32 statistics over the row, before the TF32
 * rounding of the next GEMM's operand.  Observation records and final observations hold the raw observations.
 * Everything else -- the parameters, records, sampling, log-probabilities, episode semantics and refusals -- is that of
 * mpe_rollout_policy_mlp_categorical[_episodes], with two more refusals: hidden != 64 (MPE_ERR_UNSUPPORTED, with the
 * scenario, before any pointer) and bits of net_flags above 1 or an ln_eps that is negative or not finite
 * (MPE_ERR_BAD_ARG, after the flags). */
MPE_API int mpe_rollout_policy_mappo(mpe_handle h, void *agent_pv_dev, const void *lm_p_dev, float *comm_dev,
                                     const int32_t *goal_dev, const float *const *w1_n, const float *const *b1_n,
                                     const float *const *w2_n, const float *const *b2_n, const float *const *w3_n,
                                     const float *const *b3_n, int32_t hidden, int32_t n_steps, int32_t explore,
                                     uint64_t explore_seed, uint64_t explore_epoch, uint64_t world_offset,
                                     float *const *obs_n_dev, float *rew_sum_dev, float *rew_steps_dev,
                                     float *logp_steps_dev, int32_t *const *act_index_record_n,
                                     float *const *obs_record_n, uint32_t net_flags, float ln_eps, uint8_t *done_dev,
                                     uint32_t flags, void *stream);
MPE_API int mpe_rollout_policy_mappo_episodes(
    mpe_handle h, void *agent_pv_dev, void *lm_p_dev, float *comm_dev, int32_t *goal_dev, const float *const *w1_n,
    const float *const *b1_n, const float *const *w2_n, const float *const *b2_n, const float *const *w3_n,
    const float *const *b3_n, int32_t hidden, int32_t episode_length, int32_t n_episodes, int32_t explore,
    uint64_t explore_seed, uint64_t explore_epoch, uint64_t reset_seed, uint64_t reset_epoch, uint64_t world_offset,
    float *const *obs_n_dev, float *ep_rew_dev, float *rew_steps_dev, float *logp_steps_dev,
    int32_t *const *act_index_record_n, float *const *obs_record_n, float *const *final_obs_record_n,
    uint32_t net_flags, float ln_eps, uint8_t *done_dev, uint32_t flags, void *stream);

/* MAPPO's recurrent actor (R_Actor with use_recurrent_policy, recurrent_N = 1), ONE weight set shared by every agent
 * (share_policy), hidden width 64 only: x = MAPPO's base above without its last Linear, then
 *     r = sigmoid(W_ir x + b_ir + W_hr h + b_hr),  z = sigmoid(W_iz x + b_iz + W_hz h + b_hz)
 *     n = tanh(W_in x + b_in + r * (W_hn h + b_hn)),  h' = (1 - z) * n + z * h
 *     logits = W3 LN(h') + b3
 * w_ih, w_hh are torch.nn.GRU's weight_ih_l0, weight_hh_l0 ([192][64], rows r, z, n), b_ih, b_hh its biases [192].  The
 * base folds as MAPPO's; the base's last LayerNorm is folded into w_ih, b_ih and the GRU's LayerNorm into w3, b3.
 * Built for programs whose agents all have one observation and one action size (simple, simple_spread N = 2..6,
 * simple_reference); others return MPE_ERR_UNSUPPORTED.  rnn_state_dev ([A][N][64] fp32, required) holds the hidden
 * state: read at each agent's turn and overwritten with h', so it holds the state after the last step when the call
 * ends.  The episode form starts every episode from h = 0 and never reads it.  rnn_state_record_dev ([T][A][N][64],
 * or NULL) receives the h each step's actor consumed.  Everything else is mpe_rollout_policy_mappo[_episodes]'s,
 * including the return codes and their order; a null weight counts as a null weight array. */
MPE_API int mpe_rollout_policy_gru(mpe_handle h, void *agent_pv_dev, const void *lm_p_dev, float *comm_dev,
                                   const int32_t *goal_dev, const float *w1, const float *b1, const float *w2,
                                   const float *b2, const float *w_ih, const float *b_ih, const float *w_hh,
                                   const float *b_hh, const float *w3, const float *b3, int32_t hidden, int32_t n_steps,
                                   int32_t explore, uint64_t explore_seed, uint64_t explore_epoch, uint64_t world_offset,
                                   float *const *obs_n_dev, float *rew_sum_dev, float *rew_steps_dev,
                                   float *logp_steps_dev, int32_t *const *act_index_record_n, float *const *obs_record_n,
                                   float *rnn_state_dev, float *rnn_state_record_dev, uint32_t net_flags, float ln_eps,
                                   uint8_t *done_dev, uint32_t flags, void *stream);
MPE_API int mpe_rollout_policy_gru_episodes(
    mpe_handle h, void *agent_pv_dev, void *lm_p_dev, float *comm_dev, int32_t *goal_dev, const float *w1,
    const float *b1, const float *w2, const float *b2, const float *w_ih, const float *b_ih, const float *w_hh,
    const float *b_hh, const float *w3, const float *b3, int32_t hidden, int32_t episode_length, int32_t n_episodes,
    int32_t explore, uint64_t explore_seed, uint64_t explore_epoch, uint64_t reset_seed, uint64_t reset_epoch,
    uint64_t world_offset, float *const *obs_n_dev, float *ep_rew_dev, float *rew_steps_dev, float *logp_steps_dev,
    int32_t *const *act_index_record_n, float *const *obs_record_n, float *const *final_obs_record_n,
    float *rnn_state_dev, float *rnn_state_record_dev, uint32_t net_flags, float ln_eps, uint8_t *done_dev,
    uint32_t flags, void *stream);

/* rMAPPO's separated runner: MAPPO's recurrent actor with agent i's OWN weight set (its own R_Actor), for the programs
 * whose agents observe or act differently (built for simple_speaker_listener).  The arguments are
 * mpe_rollout_policy_gru[_episodes]'s with one device pointer per agent for each of the ten folded weights (agent i's
 * W1 [64][obs_dim_i] ... W3 [act_dim_i][64], b3 [act_dim_i]), plus workspace_dev: at least
 * mpe_rollout_policy_gru_separated_workspace_bytes(h) bytes, 16-byte aligned, contents on entry irrelevant.  Every
 * call first writes each agent's TF32 fragment image into the workspace, then runs the rollout, which copies agent i's
 * image into shared memory (one TMA bulk copy) at agent i's turn of every step: every agent's weights do not fit at
 * once.  Calls that share a workspace must be ordered on one stream.  rnn_state_dev [A][N][64] and
 * rnn_state_record_dev [T][A][N][64] are agent i's h at row i, as in the shared form.  Return codes and their order are
 * mpe_rollout_policy_gru[_episodes]'s: MPE_ERR_UNSUPPORTED at the program check for a program without per-agent
 * recurrent actors or a hidden width other than 64; MPE_ERR_BAD_ARG with the null weight arrays for a null one of the
 * ten arrays, with the per-agent weight checks for a null or misaligned agent pointer, and, after the observation
 * records, for a null, not 16-byte aligned or too small workspace. */
MPE_API int mpe_rollout_policy_gru_separated(
    mpe_handle h, void *agent_pv_dev, const void *lm_p_dev, float *comm_dev, const int32_t *goal_dev,
    const float *const *w1_n, const float *const *b1_n, const float *const *w2_n, const float *const *b2_n,
    const float *const *w_ih_n, const float *const *b_ih_n, const float *const *w_hh_n, const float *const *b_hh_n,
    const float *const *w3_n, const float *const *b3_n, int32_t hidden, int32_t n_steps, int32_t explore,
    uint64_t explore_seed, uint64_t explore_epoch, uint64_t world_offset, float *const *obs_n_dev, float *rew_sum_dev,
    float *rew_steps_dev, float *logp_steps_dev, int32_t *const *act_index_record_n, float *const *obs_record_n,
    float *rnn_state_dev, float *rnn_state_record_dev, void *workspace_dev, int64_t workspace_bytes, uint32_t net_flags,
    float ln_eps, uint8_t *done_dev, uint32_t flags, void *stream);
MPE_API int mpe_rollout_policy_gru_separated_episodes(
    mpe_handle h, void *agent_pv_dev, void *lm_p_dev, float *comm_dev, int32_t *goal_dev, const float *const *w1_n,
    const float *const *b1_n, const float *const *w2_n, const float *const *b2_n, const float *const *w_ih_n,
    const float *const *b_ih_n, const float *const *w_hh_n, const float *const *b_hh_n, const float *const *w3_n,
    const float *const *b3_n, int32_t hidden, int32_t episode_length, int32_t n_episodes, int32_t explore,
    uint64_t explore_seed, uint64_t explore_epoch, uint64_t reset_seed, uint64_t reset_epoch, uint64_t world_offset,
    float *const *obs_n_dev, float *ep_rew_dev, float *rew_steps_dev, float *logp_steps_dev,
    int32_t *const *act_index_record_n, float *const *obs_record_n, float *const *final_obs_record_n,
    float *rnn_state_dev, float *rnn_state_record_dev, void *workspace_dev, int64_t workspace_bytes, uint32_t net_flags,
    float ln_eps, uint8_t *done_dev, uint32_t flags, void *stream);
/* bytes of the separated rollout's workspace: every agent's fragment image, each padded to 16 bytes (speaker_listener:
 * 120 864 + 122 912 = 243 776).  Needs no device.  MPE_ERR_BAD_ARG for a null handle, MPE_ERR_UNSUPPORTED for a
 * program without per-agent recurrent actors. */
MPE_API int64_t mpe_rollout_policy_gru_separated_workspace_bytes(mpe_handle h);

/* MAPPO's MLP actor (mpe_rollout_policy_mappo[_episodes]) with MAPPO's centralized critic (R_Critic with
 * use_centralized_V, non-recurrent, hidden width 64) evaluated in the same launch:
 *     [LN(D)] -> Linear(D, 64) -> act -> LN(64) -> Linear(64, 64) -> act -> LN(64) -> Linear(64, 1)
 * on share_obs, every agent's raw observation concatenated in agent order (D = sum of obs_dim_i), with the actor's act,
 * input LayerNorm (net_flags) and ln_eps; cw1_n .. cb3_n its folded weights (as the actor's: [64][D], [64], [64][64],
 * [64], [1][64], [1]), critic_count pointers each.  critic_count 1: one shared critic whose value is written for every
 * agent; critic_count A: agent i's own critic.  values_dev ([T][A][N] fp32, required) receives V of the state each step's
 * actors act on; final_values_dev ([A][N], in the episode form [n_episodes][A][N], required) V of the state after the
 * last step (of each episode, before its reset).  The critic changes nothing else: every other output, record and
 * state is bit-identical to mpe_rollout_policy_mappo[_episodes]'s.  Return codes and their order are MAPPO's, plus:
 * MPE_ERR_UNSUPPORTED, after the program check, for a program without the critic kernel (simple_spread N = 6,
 * simple_tag 6+2, simple_world_comm) or when critic_count critics leave no room for a warp in shared memory;
 * MPE_ERR_BAD_ARG there for a critic_count other than 1 or A, and after the recurrent actor's checks for a null or
 * misaligned critic weight or value record. */
MPE_API int mpe_rollout_policy_mappo_critic(
    mpe_handle h, void *agent_pv_dev, const void *lm_p_dev, float *comm_dev, const int32_t *goal_dev,
    const float *const *w1_n, const float *const *b1_n, const float *const *w2_n, const float *const *b2_n,
    const float *const *w3_n, const float *const *b3_n, int32_t hidden, int32_t n_steps, int32_t explore,
    uint64_t explore_seed, uint64_t explore_epoch, uint64_t world_offset, float *const *obs_n_dev, float *rew_sum_dev,
    float *rew_steps_dev, float *logp_steps_dev, int32_t *const *act_index_record_n, float *const *obs_record_n,
    uint32_t net_flags, float ln_eps, int32_t critic_count, const float *const *cw1_n, const float *const *cb1_n,
    const float *const *cw2_n, const float *const *cb2_n, const float *const *cw3_n, const float *const *cb3_n,
    float *values_dev, float *final_values_dev, uint8_t *done_dev, uint32_t flags, void *stream);
MPE_API int mpe_rollout_policy_mappo_critic_episodes(
    mpe_handle h, void *agent_pv_dev, void *lm_p_dev, float *comm_dev, int32_t *goal_dev, const float *const *w1_n,
    const float *const *b1_n, const float *const *w2_n, const float *const *b2_n, const float *const *w3_n,
    const float *const *b3_n, int32_t hidden, int32_t episode_length, int32_t n_episodes, int32_t explore,
    uint64_t explore_seed, uint64_t explore_epoch, uint64_t reset_seed, uint64_t reset_epoch, uint64_t world_offset,
    float *const *obs_n_dev, float *ep_rew_dev, float *rew_steps_dev, float *logp_steps_dev,
    int32_t *const *act_index_record_n, float *const *obs_record_n, float *const *final_obs_record_n,
    uint32_t net_flags, float ln_eps, int32_t critic_count, const float *const *cw1_n, const float *const *cb1_n,
    const float *const *cw2_n, const float *const *cb2_n, const float *const *cw3_n, const float *const *cb3_n,
    float *values_dev, float *final_values_dev, uint8_t *done_dev, uint32_t flags, void *stream);
/* MAPPO's MLP actor with IPPO's local critics (MAPPO with use_centralized_V = False) in the same launch: agent k's
 * critic is the critic above on its own raw observation, D = obs_dim_k (cw1_n[k] is [64][obs_dim_k]).  critic_count 1:
 * one shared critic evaluated once per agent on that agent's observation, which needs every obs_dim_i equal;
 * critic_count A: agent k's own critic.  values_dev[t][k][w] = V_k(o_t^k), final_values_dev as
 * mpe_rollout_policy_mappo_critic[_episodes]'s.  Parameters, semantics and return codes are
 * mpe_rollout_policy_mappo_critic[_episodes]'s, in the same order, except that MPE_ERR_UNSUPPORTED names a program
 * without these kernels (simple_tag 4+2 and 6+2, simple_world_comm) or critics that leave no room for a warp
 * (critic_count A on simple_spread N = 5 and 6), and that MPE_ERR_BAD_ARG at the critic_count check also refuses
 * critic_count 1 on a program whose agents' obs_dims differ. */
MPE_API int mpe_rollout_policy_mappo_local_critic(
    mpe_handle h, void *agent_pv_dev, const void *lm_p_dev, float *comm_dev, const int32_t *goal_dev,
    const float *const *w1_n, const float *const *b1_n, const float *const *w2_n, const float *const *b2_n,
    const float *const *w3_n, const float *const *b3_n, int32_t hidden, int32_t n_steps, int32_t explore,
    uint64_t explore_seed, uint64_t explore_epoch, uint64_t world_offset, float *const *obs_n_dev, float *rew_sum_dev,
    float *rew_steps_dev, float *logp_steps_dev, int32_t *const *act_index_record_n, float *const *obs_record_n,
    uint32_t net_flags, float ln_eps, int32_t critic_count, const float *const *cw1_n, const float *const *cb1_n,
    const float *const *cw2_n, const float *const *cb2_n, const float *const *cw3_n, const float *const *cb3_n,
    float *values_dev, float *final_values_dev, uint8_t *done_dev, uint32_t flags, void *stream);
MPE_API int mpe_rollout_policy_mappo_local_critic_episodes(
    mpe_handle h, void *agent_pv_dev, void *lm_p_dev, float *comm_dev, int32_t *goal_dev, const float *const *w1_n,
    const float *const *b1_n, const float *const *w2_n, const float *const *b2_n, const float *const *w3_n,
    const float *const *b3_n, int32_t hidden, int32_t episode_length, int32_t n_episodes, int32_t explore,
    uint64_t explore_seed, uint64_t explore_epoch, uint64_t reset_seed, uint64_t reset_epoch, uint64_t world_offset,
    float *const *obs_n_dev, float *ep_rew_dev, float *rew_steps_dev, float *logp_steps_dev,
    int32_t *const *act_index_record_n, float *const *obs_record_n, float *const *final_obs_record_n,
    uint32_t net_flags, float ln_eps, int32_t critic_count, const float *const *cw1_n, const float *const *cb1_n,
    const float *const *cw2_n, const float *const *cb2_n, const float *const *cw3_n, const float *const *cb3_n,
    float *values_dev, float *final_values_dev, uint8_t *done_dev, uint32_t flags, void *stream);

/* rMAPPO's recurrent centralized critic (R_Critic with use_recurrent_policy, recurrent_N = 1, use_centralized_V,
 * hidden width 64), ONE weight set shared by every agent, run as a kernel of its own after
 * mpe_rollout_policy_gru[_episodes] on the same stream, over that rollout's observation records:
 *     x = [LN(D)] -> Linear(D, 64) -> act -> LN(64) -> Linear(64, 64) -> act -> LN(64),  h' = GRU(x, h)
 *     V = w3 LN(h') + b3
 * on share_obs, every agent's raw observation concatenated in agent order (D = sum of obs_dim_i), folded as
 * mpe_rollout_policy_gru's actor (w1 [64][D], w3 [1][64], b3 [1]; the others as the actor's).  obs_record_n[i]
 * ([T][N][obs_dim_i]) is the rollout's observation record, final_obs_n[i] ([E][N][obs_dim_i]) its final observations:
 * the returned observations for one episode (E = 1), the final-observation record in the episode form.  Per step t:
 * values_dev[t][a][w] = V (the same for every agent a, [T][A][N]) and h = h'.  episode_length L = 0: one episode of
 * n_steps, h starting from rnn_state_dev ([N][64], read) and final_values_dev[0] ([1][A][N]) = V(final_obs_n, h') after
 * the last step.  L > 0: n_steps / L = E episodes, each starting from h = 0 (rnn_state_dev is not read), and
 * final_values_dev[e] ([E][A][N]) is V of episode e's final observation, taken from the h after its last step.
 * rnn_state_dev receives the h after the last step in both forms; rnn_state_record_dev ([T][N][64], or NULL) the h
 * each step consumed.  Checked in this order: MPE_ERR_BAD_ARG for a null handle or n_steps < 0; MPE_ERR_NO_DEVICE;
 * MPE_ERR_UNSUPPORTED for a program without the kernel (built for simple, simple_spread N = 2..6 and
 * simple_reference); MPE_ERR_BAD_ARG for episode_length < 0, or > 0 without dividing n_steps >= 1; for unknown
 * net_flags or an eps that is negative, NaN or infinite; for a null or misaligned weight, state, record, value array,
 * observation array or agent observation pointer (values_dev and obs_record_n may be null when n_steps is 0). */
MPE_API int mpe_critic_gru(mpe_handle h, const float *const *obs_record_n, const float *const *final_obs_n,
                           int32_t n_steps, int32_t episode_length, const float *w1, const float *b1, const float *w2,
                           const float *b2, const float *w_ih, const float *b_ih, const float *w_hh,
                           const float *b_hh, const float *w3, const float *b3, float *rnn_state_dev,
                           float *rnn_state_record_dev, float *values_dev, float *final_values_dev,
                           uint32_t net_flags, float ln_eps, void *stream);
/* rMAPPO's separated runner's critics: agent k's own recurrent critic (R_Critic on share_obs, k = 0 .. A-1), its ten
 * folded weights at w*_n[k], all A in one launch.  As mpe_critic_gru but: rnn_state_dev is [A][N][64] (critic k's h at
 * row k), rnn_state_record_dev [n_steps][A][N][64], and values_dev / final_values_dev receive critic k's value in agent
 * k's row only.  Return codes and their order are mpe_critic_gru's; MPE_ERR_UNSUPPORTED for a program without
 * per-agent recurrent actors, MPE_ERR_BAD_ARG at the weight check for a null array or a null or misaligned agent
 * pointer. */
MPE_API int mpe_critic_gru_separated(mpe_handle h, const float *const *obs_record_n, const float *const *final_obs_n,
                                     int32_t n_steps, int32_t episode_length, const float *const *w1_n,
                                     const float *const *b1_n, const float *const *w2_n, const float *const *b2_n,
                                     const float *const *w_ih_n, const float *const *b_ih_n, const float *const *w_hh_n,
                                     const float *const *b_hh_n, const float *const *w3_n, const float *const *b3_n,
                                     float *rnn_state_dev, float *rnn_state_record_dev, float *values_dev,
                                     float *final_values_dev, uint32_t net_flags, float ln_eps, void *stream);
/* rIPPO's recurrent local critic (R_Critic with use_centralized_V = False): ONE weight set shared by every agent, run on
 * agent k's own observation record for k = 0 .. A-1 in one launch, w1 [64][obs_dim] (every agent observes alike on
 * these programs).  As mpe_critic_gru but: agent k's critic reads obs_record_n[k] and final_obs_n[k] only,
 * rnn_state_dev is [A][N][64] (agent k's h at row k), rnn_state_record_dev [n_steps][A][N][64], and values_dev[t][k]
 * and final_values_dev[e][k] receive agent k's own value.  Return codes and their order are mpe_critic_gru's
 * (MPE_ERR_UNSUPPORTED: built for simple, simple_spread N = 2..6 and simple_reference). */
MPE_API int mpe_critic_gru_local(mpe_handle h, const float *const *obs_record_n, const float *const *final_obs_n,
                                 int32_t n_steps, int32_t episode_length, const float *w1, const float *b1,
                                 const float *w2, const float *b2, const float *w_ih, const float *b_ih,
                                 const float *w_hh, const float *b_hh, const float *w3, const float *b3,
                                 float *rnn_state_dev, float *rnn_state_record_dev, float *values_dev,
                                 float *final_values_dev, uint32_t net_flags, float ln_eps, void *stream);

/* flags of mpe_gae */
enum mpe_gae_flags {
    MPE_GAE_BOOTSTRAP = 1,              /* an episode end is a time-limit truncation: continue with gamma * V(final) */
    MPE_GAE_NORMALIZE = 2,              /* normalise the advantages over all T * A * N entries (PPO's update step) */
    MPE_GAE_PER_AGENT_VALUE_NORM = 4    /* value_norm_dev holds one (mean, std) row per agent, [A][2] */
};

/* MAPPO's GAE advantages and returns (SharedReplayBuffer.compute_returns with use_gae) over a finished buffer, on the
 * device, for any handle: only its A and N are used.  rewards_dev, values_dev, returns_dev and advantages_dev are
 * float32 [T][A][N] (T = n_steps); final_values_dev [E][A][N], E = n_steps / L.  episode_length L = 0 is one episode
 * of n_steps; L > 0 makes episode e steps e*L .. e*L + L - 1.  value_norm_dev (NULL: no ValueNorm) holds float32
 * (mean, std), [2] for every agent or [A][2] with MPE_GAE_PER_AGENT_VALUE_NORM; every value v is denormalised as
 * dv = v * std + mean (else dv = v).  It is read on the device: the call never synchronises with the host and can be
 * captured in a CUDA graph.  Per column (agent, world), t running backwards inside each episode:
 *     last   = t is the last step of its episode
 *     next   = last ? (MPE_GAE_BOOTSTRAP ? dv(final_values[e]) : 0) : dv[t + 1]
 *     carry  = last ? 0 : gae[t + 1]
 *     delta  = (r[t] + gamma * next) - dv[t]
 *     gae[t] = delta + (gamma * gae_lambda) * carry      gamma * gae_lambda: one fp32 product
 *     ret[t] = gae[t] + dv[t]
 * in fp32, every operation rounded to nearest in exactly this order, with no fused multiply-add.  returns_dev
 * receives ret, advantages_dev gae.  MPE_GAE_NORMALIZE replaces every advantage a by
 * float((double(a) - mean) / (std + 1e-5)), mean and std (population) over all T * A * N advantages, summed in fp64
 * per scan block and combined in a fixed order: two calls give the same bits.  (mean, std) is then left as two
 * doubles at the start of the workspace.  workspace_dev (8-byte aligned, at least mpe_gae_workspace_bytes(h) bytes,
 * contents on entry irrelevant) is needed only with MPE_GAE_NORMALIZE and may be NULL without it; calls that share a
 * workspace must be ordered on one stream.  Outputs must not overlap the inputs, each other or the workspace.
 * Checked in this order: MPE_ERR_BAD_ARG for a null handle or n_steps < 1; MPE_ERR_NO_DEVICE; MPE_ERR_BAD_ARG for
 * episode_length < 0 or not dividing n_steps; for gamma or gae_lambda outside [0, 1] or not finite; for unknown flag
 * bits; for a null or misaligned (not 4-byte aligned) rewards, values, returns or advantages array, a null or
 * misaligned final_values_dev with MPE_GAE_BOOTSTRAP (without it, it is not read and may be NULL), a misaligned
 * value_norm_dev or a null one with MPE_GAE_PER_AGENT_VALUE_NORM, and, with MPE_GAE_NORMALIZE, a null, not 8-byte
 * aligned or too small workspace. */
MPE_API int mpe_gae(mpe_handle h, const float *rewards_dev, const float *values_dev, const float *final_values_dev,
                    int32_t n_steps, int32_t episode_length, float gamma, float gae_lambda, uint32_t flags,
                    const float *value_norm_dev, float *returns_dev, float *advantages_dev, void *workspace_dev,
                    int64_t workspace_bytes, void *stream);
/* bytes of mpe_gae's workspace for this handle (32 + 16 per 128 columns of A * N), or MPE_ERR_BAD_ARG for a null
 * handle */
MPE_API int64_t mpe_gae_workspace_bytes(mpe_handle h);

/* Same step for a caller that holds HOST buffers (what the reference's callers hold):
 * act_n_host[i] -> (async H2D into act_n_dev[i]) -> mpe_step -> (async D2H) obs_n_host[i],
 * rew_host, done_host, all ordered on `stream`.  Host buffers should be pinned for the copies
 * to be asynchronous.  The caller synchronises the stream before reading the outputs.
 * Large batches are cut into MPE_B200_HOST_CHUNKS (default 4) world ranges that alternate
 * between two library-owned streams forked from / joined to `stream`, so that the upload + step of one range
 * overlaps the download of the previous one (full-duplex PCIe).  Pipelining starts at MPE_B200_HOST_CHUNK_MIN worlds (default 262144: below that the
 * extra copy calls cost more than the overlap gains on PCIe Gen5). */
MPE_API int mpe_step_host(mpe_handle h, void *agent_pv_dev, const void *lm_p_dev, float *comm_dev,
                  const int32_t *goal_dev, const float *const *act_n_host, float *const *act_n_dev,
                  float *const *obs_n_dev, float *rew_dev, uint8_t *done_dev, float *info_dev,
                  float *const *obs_n_host, float *rew_host, uint8_t *done_host, float *info_host,
                  uint32_t flags, void *stream);

/* ---- diagnostics --------------------------------------------------------------------------- */
MPE_API const char *mpe_strerror(int err);
MPE_API const char *mpe_last_cuda_error(void);  /* text of the last CUDA failure on this thread */
MPE_API int mpe_abi_version(void);
MPE_API int64_t mpe_kernel_launches(void);      /* kernels launched by this library so far (process-wide) */
/* Measurement aid (bench.py "size-matched streaming ceiling"): one launch of a pure streaming kernel that reads
 * read_bytes from src_dev and then writes write_bytes to dst_dev (both 16-byte aligned) with `threads` threads,
 * through the same launch path as mpe_step.  Not counted by mpe_kernel_launches; computes nothing. */
MPE_API int mpe_probe_stream(int device, const void *src_dev, int64_t read_bytes, void *dst_dev, int64_t write_bytes,
                             int64_t threads, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* MPE_B200_H */
