"""MultiAgentEnv: the gym-style adapter over a (batched) World
(reference: multiagent/environment.py:12-263).

Same constructor, attributes and `step` / `reset` contract as the reference.  The per-agent
Python loops of the reference's `step` (`_set_action` -> `world.step()` -> observation / reward /
done / info callbacks -> shared-reward sum, environment.py:80-104) are ONE launch of the fused
sm_90a kernel (`mpe_step`) over all worlds of the batch.

Calling conventions
  scalar mode  (world.num_envs is None; what `make_env(name)` gives): identical to the reference --
      `action_n[i]` is a 1-D array, `obs_n[i]` a float64 ndarray, `reward_n[i]` a float,
      `done_n[i]` a bool, `info_n == {'n': [...]}`.
  batched mode (world.num_envs = N): `action_n[i]` is `[N, act_dim_i]`; CUDA tensors in ->
      CUDA tensors out (`obs_n[i]: [N, obs_dim_i]`, `reward_n[i]: [N]`, `done_n[i]: [N] bool`);
      NumPy arrays / CPU tensors in -> the step runs through pinned staging (`mpe_step_host`) and
      NumPy arrays / CPU tensors come back.
"""
import numpy as np

from . import _lib
from .multi_discrete import MultiDiscrete
from .scenario import NativeScenario
from . import spaces

try:  # pragma: no cover
    from gym import Env as _Env
except Exception:  # noqa: BLE001
    class _Env(object):
        pass


class MultiAgentEnv(_Env):
    metadata = {'render.modes': ['human', 'rgb_array']}

    def __init__(self, world, reset_callback=None, reward_callback=None,
                 observation_callback=None, info_callback=None,
                 done_callback=None, shared_viewer=True):
        self.world = world
        self.agents = self.world.policy_agents
        self.n = len(world.policy_agents)
        self.reset_callback = reset_callback
        self.reward_callback = reward_callback
        self.observation_callback = observation_callback
        self.info_callback = info_callback
        self.done_callback = done_callback
        # environment parameters (environment.py:28-36)
        self.discrete_action_space = True
        self.discrete_action_input = False
        self.force_discrete_action = world.discrete_action if hasattr(world, 'discrete_action') else False
        self.shared_reward = world.collaborative if hasattr(world, 'collaborative') else False
        self.time = 0
        #: batched mode: hand out views of the library's persistent result buffers instead of freshly allocated
        #: tensors / arrays.  CUDA callers: every step writes the same device slab (results are overwritten by the
        #: next step).  Host callers: results are views of two flip-flopped pinned slabs (valid until the
        #: next-but-one step).  Default False = the reference's ownership: every step returns fresh arrays.
        self.reuse_buffers = False
        #: exploration epoch of rollout_policy(..., explore_seed=s): part of the noise counter, advanced by one per
        #: exploring call, so consecutive calls draw fresh noise and a new env with the same seed replays the sequence
        self.explore_epoch = 0

        self._custom = (getattr(world, "native_program", None) == "custom")
        if self._custom and not world.batched:
            raise NotImplementedError("user scenarios (TorchScenario) run in batched mode only: pass num_envs")
        for name, cb in (("reward_callback", reward_callback), ("observation_callback", observation_callback)):
            owner = getattr(cb, "__self__", None)
            if cb is not None and not self._custom and not isinstance(owner, NativeScenario):
                raise NotImplementedError(
                    "%s is an arbitrary Python callable; only scenarios with a compiled sm_90a program "
                    "(subclasses of NativeScenario) can be stepped, and there is no CPU fallback" % name)
        self._native_info = info_callback is not None and isinstance(getattr(info_callback, "__self__", None),
                                                                     NativeScenario)
        shapes = world.native_shapes()   # validates the descriptor; works without a GPU
        if shapes.n_agents != self.n:
            raise ValueError("native program agent count mismatch")

        # configure spaces (environment.py:39-70)
        self.action_space = []
        self.observation_space = []
        for i, agent in enumerate(self.agents):
            total_action_space = []
            if agent.movable:
                total_action_space.append(spaces.Discrete(world.dim_p * 2 + 1))
            if not agent.silent:
                total_action_space.append(spaces.Discrete(world.dim_c))
            if len(total_action_space) > 1:
                self.action_space.append(MultiDiscrete([[0, sp.n - 1] for sp in total_action_space]))
            else:
                self.action_space.append(total_action_space[0])
            if self._custom:   # as the reference does (environment.py:68): ask the callback (binds the batch: needs the GPU)
                world.bind()
                obs_dim = int(observation_callback(agent, world).shape[-1])
            else:
                obs_dim = shapes.obs_dims[i]
            self.observation_space.append(spaces.Box(low=-np.inf, high=+np.inf, shape=(obs_dim,), dtype=np.float32))
        self._act_dims = list(shapes.act_dims)
        self._sub_sizes = [([5] if a.movable else []) + ([world.dim_c] if not a.silent else []) for a in self.agents]

        # rendering (headless; attributes kept for API compatibility)
        self.shared_viewer = shared_viewer
        self.viewers = [None] if shared_viewer else [None] * self.n
        self._reset_render()

    # ------------------------------------------------------------------------------------------
    def _flags(self):
        f = 0
        if self.shared_reward:
            f |= _lib.FLAG_SHARED_REWARD
        if self.force_discrete_action:
            f |= _lib.FLAG_FORCE_DISCRETE_ACTION
        if not self.discrete_action_space:
            raise NotImplementedError("discrete_action_space=False is not supported (hard-coded True in the "
                                      "reference, environment.py:29)")
        return f

    def _index_tensors(self, action_n, nw):
        """discrete_action_input (environment.py:161-167,185-187): the kernel decodes integer sub-actions itself
        (MPE_FLAG_DISCRETE_ACTION_INPUT): action_n[i] becomes int32 [N, n_sub_i] on the device -- a no-op for a
        contiguous int32 CUDA tensor of that shape; other dtypes / host arrays are converted / uploaded here.
        Movement index 0 = none, 1 = -x, 2 = +x, 3 = -y, 4 = +y; utterance index k -> one-hot(k)."""
        import torch
        N = self.world.batch_size
        out = []
        for i, a in enumerate(action_n):
            nsub = len(self._sub_sizes[i])
            if not torch.is_tensor(a):
                a = torch.as_tensor(np.ascontiguousarray(np.asarray(a)).astype(np.int32, copy=False))
            if a.numel() != N * nsub:
                raise ValueError("action_n[%d] must hold %d x %d integer sub-actions, got shape %s"
                                 % (i, N, nsub, tuple(a.shape)))
            if a.device != nw.device or a.dtype != torch.int32:
                a = a.to(device=nw.device, dtype=torch.int32)
            out.append(a.reshape(N, nsub).contiguous())
        return out

    def _step_discrete(self, action_n, nw, flags):
        world = self.world
        on_device = all(hasattr(a, "is_cuda") and a.is_cuda for a in action_n)
        as_numpy = not any(hasattr(a, "dim") for a in action_n)
        idx = self._index_tensors(action_n, nw)
        flags |= _lib.FLAG_DISCRETE_ACTION_INPUT
        if self._custom:
            return self._step_custom(idx, nw, flags)
        out = nw.out if (self.reuse_buffers or not world.batched) else nw.new_outputs()
        nw.step(_lib.ptr_array([t.data_ptr() for t in idx]), out, flags, with_info=self._native_info)
        self._last_out = out
        world._obs_valid = False
        if not world.batched:
            return self._pack_scalar(nw, out)
        obs_n, reward_n, done_n, info_n = self._pack_batched(nw, out)
        if not on_device:     # host callers get host results back
            obs_n, reward_n, done_n = ([t.cpu() for t in x] for x in (obs_n, reward_n, done_n))
            if as_numpy:
                obs_n, reward_n, done_n = ([t.numpy() for t in x] for x in (obs_n, reward_n, done_n))
        return obs_n, reward_n, done_n, info_n

    def step(self, action_n):
        world = self.world
        nw = world.bind()
        self.agents = world.policy_agents
        if len(action_n) != self.n:
            raise ValueError("expected %d actions, got %d" % (self.n, len(action_n)))
        flags = self._flags()
        if self.discrete_action_input:
            return self._step_discrete(action_n, nw, flags)
        if self._custom:
            return self._step_custom(action_n, nw, flags)
        if not world.batched and not any(hasattr(a, "dim") for a in action_n):
            # scalar convention fast path: NumPy in, NumPy out, no tensor objects created per step
            hs = nw.host_staging()
            for i, a in enumerate(action_n):
                np.copyto(hs["host_act_np"][i][0], np.asarray(a, dtype=np.float32).reshape(-1))
            hout = nw.step_host(hs["host_act_ptrs"], flags, with_info=self._native_info)
            nw.torch.cuda.current_stream(nw.device).synchronize()
            self._last_out = hout
            world._obs_valid = False
            return self._pack_scalar(nw, hout)
        mode, payload = self._classify(action_n, nw)
        if mode == "cuda":
            out = nw.out if self.reuse_buffers else nw.new_outputs()
            nw.step(_lib.ptr_array([t.data_ptr() for t in payload]), out, flags, with_info=self._native_info)
            self._last_out = out
            world._obs_valid = False
            if not world.batched:     # scalar convention with device-side inputs (e.g. discrete_action_input)
                return self._pack_scalar(nw, out)
            return self._pack_batched(nw, out)
        # host callers: pinned staging -> mpe_step_host -> pinned outputs
        hs = nw.host_staging()
        ptrs = []
        for i, a in enumerate(payload):
            if mode == "pinned":
                ptrs.append(a.data_ptr())
            else:
                hs["host_act"][i].copy_(a if hasattr(a, "dim") else self._to_cpu_tensor(a, i))
                ptrs.append(hs["host_act"][i].data_ptr())
        hout = nw.step_host(_lib.ptr_array(ptrs), flags, with_info=self._native_info)
        nw.torch.cuda.current_stream(nw.device).synchronize()
        self._last_out = hout
        world._obs_valid = False
        if not world.batched:
            return self._pack_scalar(nw, hout)
        as_numpy = not hasattr(action_n[0], "dim")
        return self._pack_batched(nw, hout, as_numpy=as_numpy)

    # ---- K-step open-loop rollout (batch extension; SURVEY.md 8(f) rank 3) -------------------------
    def rollout(self, action_seq_n, per_step_rewards=False):
        """T consecutive `step` calls on pre-generated actions in ONE kernel launch (mpe_rollout): the loop of
        bin/interactive.py:27-39 when the actions are known in advance (recorded trajectories, CEM / MPPI candidate
        sequences).  action_seq_n[i]: float32 CUDA tensor [T, N, act_dim_i].  Returns (obs_n, reward_sum_n, done_n,
        info_n) for the state after the last step -- reward_sum_n[i] is the sum over the T steps, bit-equal to calling
        `step` T times and adding the rewards in order -- plus, with per_step_rewards=True, a fifth item: the [T, n, N]
        tensor of every step's rewards.  Batched CUDA mode only."""
        import torch
        world = self.world
        if not world.batched:
            raise ValueError("rollout needs a batched env (make_env(..., num_envs=N))")
        if self._custom:
            raise NotImplementedError("rollout is not available for user scenarios (TorchScenario)")
        if self.discrete_action_input:
            raise NotImplementedError("rollout takes action vectors, not integer actions")
        if len(action_seq_n) != self.n:
            raise ValueError("expected %d action sequences, got %d" % (self.n, len(action_seq_n)))
        nw = world.bind()
        N = nw.n_env
        T = int(action_seq_n[0].shape[0])
        seqs = []
        for i, a in enumerate(action_seq_n):
            if not (torch.is_tensor(a) and a.is_cuda and a.device == nw.device):
                raise ValueError("action_seq_n[%d] must be a CUDA tensor on %s" % (i, nw.device))
            if tuple(a.shape) != (T, N, self._act_dims[i]):
                raise ValueError("action_seq_n[%d] must have shape (%d, %d, %d), got %s"
                                 % (i, T, N, self._act_dims[i], tuple(a.shape)))
            if a.dtype != torch.float32 or not a.is_contiguous():
                a = a.to(torch.float32).contiguous()
            seqs.append(a)
        out = nw.out if self.reuse_buffers else nw.new_outputs()
        rew_steps = torch.empty((T, self.n, N), dtype=torch.float32, device=nw.device) if per_step_rewards else None
        nw.rollout(_lib.ptr_array([t.data_ptr() for t in seqs]), T, out, self._flags(), rew_steps)
        self._last_out = out
        world._obs_valid = False
        obs_n, reward_n, done_n = list(out.obs), list(out.rew_list), list(out.done_list)
        info_n = {'n': [{} for _ in range(self.n)]}
        if per_step_rewards:
            return obs_n, reward_n, done_n, info_n, rew_steps
        return obs_n, reward_n, done_n, info_n

    def rollout_policy(self, policies, n_steps, record_actions=False, per_step_rewards=False, record_observations=False,
                       explore_seed=None, episode_length=None, action_mode="softmax", record_log_probs=False,
                       rnn_states=None, record_rnn_states=False, critic=None, critic_rnn_states=None,
                       record_critic_rnn_states=False, centralized_critic=True):
        """T closed-loop steps in ONE kernel launch with the actors inside the kernel.

        One hidden layer (mpe_rollout_policy, fp32): agent i acts with softmax(W2_i relu(W1_i obs_i + b1_i) + b2_i).
        policies[i] is a `torch.nn.Sequential(Linear(obs_dim_i, H), ReLU(), Linear(H, 5))` or the tuple (W1 [H, obs_dim_i],
        b1 [H], W2 [5, H], b2 [5]) in torch's Linear layout, H = 32 or 64.

        Two hidden layers, MADDPG's actor (mpe_rollout_policy_mlp, TF32 tensor cores): policies[i] is a
        `torch.nn.Sequential(Linear(obs_dim_i, H), ReLU(), Linear(H, H), ReLU(), Linear(H, act_dim_i))` or the tuple
        (W1, b1, W2, b2, W3, b3), H = 32 or 64.  The act_dim_i outputs split into the agent's action sub-spaces as the
        action vector does -- 5 movement logits if it is movable, then dim_c utterance logits if it speaks -- and the
        action is one softmax per sub-space (MADDPG's SoftMultiCategoricalPd).  An utterance becomes the world's comm
        state after the step, so the other agents observe it from the next step on.  explore_seed (an int) makes every
        agent act with the Gumbel-softmax sample softmax(logits - log(-log u)) per sub-space instead; the noise is keyed
        by (explore_seed, self.explore_epoch, global world index, step, agent) and self.explore_epoch advances by one per
        exploring call.  record_observations=True returns extras["observations"], a list of [T, N, obs_dim_i] tensors:
        the observation agent i acted on at each step.  Both options need the two-hidden-layer actor.  Built for simple,
        simple_spread N=2 to 6, simple_tag 3+1, 1+1, 2+1, 4+2 and 6+2 (3 landmarks), simple_speaker_listener,
        simple_reference, simple_crypto, simple_adversary (3 or 4 agents) and simple_push (2 agents); other programs
        (simple_world_comm) raise MpeError.

        Returns (obs_n, reward_sum_n, done_n, info_n, extras) for the state after the last step; extras["actions"]
        (record_actions) is a list of [T, N, act_dim_i] tensors with the actions taken ([T, N, 5] for the one-hidden-layer
        actor), extras["rewards"] (per_step_rewards) a [T, n, N] tensor.  World state lives in registers for all T steps.
        Batched CUDA mode.  The one-hidden-layer actor needs a scenario whose agents all move and are silent and whose
        program was built with that kernel (simple, simple_spread N=3, simple_tag 3+1) -- anything else raises.

        episode_length=L (two-hidden-layer actor only) collects E = n_steps / L whole MADDPG episodes in the one launch,
        resetting every world inside the kernel after each episode.  Bit for bit the same as E calls
        rollout_policy(policies, L, ...) each followed by env.reset(): episode e explores with epoch explore_epoch + e
        (its step counter restarts at 0; explore_epoch advances by E when exploring), and the reset after it draws what
        that reset() would draw (the world's reset epoch advances by E).  Records span all n_steps steps (global step
        e * L + t).  reward_sum_n[i] is [E, N], the return of every episode; obs_n holds the observations of the freshly
        reset state, done_n is all False, and with record_observations extras["final_observations"] is a list of
        [E, N, obs_dim_i] tensors: the observation after the last step of each episode, before its reset (the next
        observation of the terminal transition).  n_steps must be a positive multiple of L (else ValueError).

        action_mode="categorical" (two-hidden-layer actor only; the default "softmax" is everything above) collects
        policy-gradient (PPO, A2C) experience: per sub-space the agent takes k = argmax(logits - log(-log u)) when
        exploring -- a categorical sample, the arg-max of the Gumbel-softmax sample the default mode would take from the
        same state, seed and epoch -- or k = argmax(logits) without explore_seed, the lowest index winning ties, and
        applies the one-hot vector of k, exactly as env.step applies that float vector.  extras["actions"]
        (record_actions) is then a list of int32 [T, N, n_sub_i] tensors, n_sub_i the agent's number of sub-spaces (1,
        or 2 for a movable speaker: movement, then utterance).  k is the position in the logit segment, i.e. the one-hot
        convention: movement index 1 is +x.  It is NOT the code env.discrete_action_input takes (there 1 is -x), so
        replay the indices as one-hot vectors, never through discrete_action_input.  record_log_probs=True returns
        extras["log_probs"], a float32 [T, n, N] tensor: the sum over the agent's sub-spaces of
        log_softmax(logits)[k] on the logits the kernel acted with (Categorical(logits).log_prob(k), the behaviour
        policy's term of PPO's ratio), else None.  Returns, observations, episode_length and both epochs behave as in
        the default mode.  An unknown action_mode, or record_log_probs in the default mode, raises ValueError; the
        one-hidden-layer actor raises NotImplementedError.

        MAPPO's MLP actor (mpe_rollout_policy_mappo, action_mode="categorical" only): policies[i] is an
        `nn.Sequential([LayerNorm(obs_dim_i)], Linear(obs_dim_i, 64), Act, LayerNorm(64), Linear(64, 64), Act,
        LayerNorm(64), Linear(64, act_dim_i))` -- MAPPO's MLPBase (layer_N = 1, the optional input LayerNorm being
        use_feature_normalization) and its categorical head -- with Act = ReLU() or Tanh(), the same everywhere, and one
        LayerNorm eps for all.  One module object may serve all agents (share_policy).  Any policy with a LayerNorm takes
        this path, and mappo_actor_params checks the layer list (ValueError).  Each LayerNorm's affine is folded into the
        next Linear (float64, then float32); the kernel normalises with fp32 statistics and TF32 GEMM operands.  Records,
        extras, sampling, log-probabilities and episodes are those of the categorical mode above; observation records and
        final observations hold the raw observations (before the input LayerNorm).  action_mode="softmax" and a hidden
        width other than 64 raise NotImplementedError.

        MAPPO's recurrent actor (mpe_rollout_policy_gru, action_mode="categorical" only; rMAPPO with recurrent_N = 1 and
        share_policy): policies is [actor] * n, ONE tuple (base, gru, norm, head) for every agent -- base the MAPPO
        actor above without its last Linear, gru an nn.GRU(64, 64), norm a LayerNorm(64), head a Linear(64, act_dim);
        rmappo_actor_params checks it (ValueError) and folds it.  Any policy tuple holding an nn.GRU takes this path;
        distinct per-agent tuples raise NotImplementedError.  Built for simple, simple_spread N = 2..6 and
        simple_reference (every other program raises MpeError before anything runs).  Per step the logits are
        head(norm(h')), h' = gru(base(obs), h), h carried across steps.  rnn_states: the initial hidden state, a float32
        CUDA tensor [n, N, 64] on the env's device, read and never written (None: zeros); it cannot be combined with
        episode_length, whose episodes each start from h = 0 (MAPPO's mask after done).  extras["final_rnn_states"] is a
        new [n, N, 64] tensor: h after the last step (of the last episode, before its reset), what the next call's
        rnn_states continues from.  record_rnn_states=True returns extras["rnn_states"], a float32 [T, n, N, 64] tensor
        of the h each step's actor consumed (MAPPO's buffer rnn_states[t]; zero at every episode's first step), else
        None -- T * n * N * 256 bytes.  Records, sampling, log-probabilities, episodes and epochs are the categorical
        mode's.  rnn_states or record_rnn_states with any other actor raise ValueError.

        Per-agent recurrent actors (mpe_rollout_policy_gru_separated, rMAPPO's separated runner): on a program whose
        agents observe or act differently -- built for simple_speaker_listener -- distinct tuples give every agent its
        own (base, gru, norm, head), each of the form above for its own obs_dim_i and act_dim_i and folded by
        rmappo_actor_params([policies[i]], [obs_dim_i], [act_dim_i]) (ValueError naming the agent); the activation,
        input LayerNorm and eps must be the same for all (ValueError).  rnn_states, the records, extras and episodes are
        the shared actor's, row i being agent i's h.  Every agent's weights do not fit in shared memory at once, so the
        call first writes each agent's TF32 fragment image to a workspace and the kernel copies agent i's into shared
        memory at its turn of every step.  On any other program distinct tuples keep the shared actor's refusal (one
        shared tuple on speaker_listener raises MpeError).  Every refusal happens before the world is bound.

        critic (MAPPO's MLP actor only, mpe_rollout_policy_mappo_critic[_episodes]) evaluates MAPPO's centralized critic
        in the same launch: R_Critic with use_centralized_V and no recurrence, `nn.Sequential([LayerNorm(D)], Linear(D,
        64), Act, LayerNorm(64), Linear(64, 64), Act, LayerNorm(64), Linear(64, 1))`, whose input is share_obs -- every
        agent's raw observation concatenated in agent order, D = sum of obs_dim_i.  Its Act, input LayerNorm and eps
        must be the actors' (ValueError); mappo_critic_params checks and folds it as the actor is folded.  Pass one
        module (or [critic] * n, the same object: share_policy), whose value is computed once per world and step and
        written for every agent, or a list of n distinct modules (per-agent critics, each evaluating the same input).
        extras["values"] is then a float32 [T, n, N] tensor, V of the observations step t's actors acted on (MAPPO's
        value_preds[t]), and extras["final_values"] a float32 [n, N] tensor, V after the last step (MAPPO's next_value);
        with episode_length it is [E, n, N], V of each episode's final observation, before its reset.  Everything else
        is bit-identical to the same call without a critic.  A critic with any other actor or with action_mode="softmax"
        raises NotImplementedError, a malformed one or a list of length other than 1 or n ValueError.  simple_spread N=6
        and simple_tag 6+2 have no critic kernel, and per-agent critics do not fit in shared memory next to the actors
        for simple_spread N=4 and 5, simple_tag 3+1 and 4+2 and simple_adversary with 4 agents: those raise MpeError
        before anything runs.

        critic with MAPPO's recurrent actor (mpe_critic_gru, rMAPPO) evaluates rMAPPO's recurrent centralized critic,
        R_Critic with recurrent_N = 1: ONE tuple (base, gru, norm, v_out), or [critic] * n (the same object) -- base
        MAPPO's MLPBase on share_obs (nn.Sequential([LayerNorm(D)], Linear(D, 64), Act, LayerNorm(64), Linear(64, 64),
        Act, LayerNorm(64))), gru an nn.GRU(64, 64), norm a LayerNorm(64), v_out a Linear(64, 1).  rmappo_critic_params
        checks and folds it as the recurrent actor is folded; its Act, input LayerNorm and eps must be the actor's
        (ValueError).  Per step t, h' = gru(base(share_obs_t), h), extras["values"][t] = v_out(norm(h')) (float32 [T, n,
        N], the same value for every agent) and h = h'; extras["final_values"] ([n, N], with episode_length [E, n, N])
        is the same formula once more on the observation after the last step (of each episode, before its reset) with
        the carried h.  critic_rnn_states: the critic's initial h, a float32 CUDA tensor [N, 64] on the env's device,
        read and never written (None: zeros; not with episode_length, whose episodes each start from h = 0).  A shared
        critic's MAPPO buffer rnn_states_critic[:, a] is the same for every agent a: pass its slice [:, 0].
        extras["final_critic_rnn_states"] is a new [N, 64] tensor, h after the last step (of the last episode), what
        the next call's critic_rnn_states continues from; record_critic_rnn_states=True returns
        extras["critic_rnn_states"], a float32 [T, N, 64] tensor of the h each step's critic consumed (zero at every
        episode's first step), else None.  The critic runs as a second kernel on the same stream, after the rollout,
        over the rollout's observation records: without record_observations they are scratch, T * N * D * 4 bytes
        (1.4 GB for simple_spread N=6 at 65 536 worlds and T = 25), and extras["observations"] stays None.  Everything
        else is bit-identical to the same call without a critic.  A recurrent critic with any other actor, an
        nn.Sequential critic with the recurrent actor (rMAPPO pairs the actor's and the critic's recurrence) and
        distinct per-agent recurrent critics raise NotImplementedError; critic_rnn_states or record_critic_rnn_states
        without a recurrent critic raise ValueError.  With per-agent recurrent actors the critic is a list of n recurrent
        tuples, one per agent (mpe_critic_gru_separated, the separated runner's R_Critic per agent on share_obs), each
        folded by rmappo_critic_params: agent k's values and final values come from critic k, critic_rnn_states and
        extras["final_critic_rnn_states"] are [n, N, 64] and extras["critic_rnn_states"] [T, n, N, 64] (MAPPO's
        separated rnn_states_critic); a single tuple or a list of another length raises ValueError.

        centralized_critic=False selects IPPO's local critics (MAPPO with use_centralized_V=False, share_obs = obs): every
        critic above reads agent k's own raw observation instead of share_obs, its input width is obs_dim_k, and
        nothing else changes -- extras keep their names and shapes and compute_gae takes them as they are.
          - With MAPPO's MLP actor (mpe_rollout_policy_mappo_local_critic[_episodes]): the critic is
            nn.Sequential([LayerNorm(obs_dim_k)], Linear(obs_dim_k, 64), Act, LayerNorm(64), Linear(64, 64), Act,
            LayerNorm(64), Linear(64, 1)), folded by mappo_actor_params on [obs_dim_k].  One module (or [critic] * n)
            is one shared critic evaluated on every agent's observation, which needs every obs_dim_i equal (simple,
            simple_spread, simple_reference); n distinct modules give agent k its own.  extras["values"][t, k] =
            V_k(obs_k at step t).  simple_tag 4+2 and 6+2 have no kernel, and n per-agent critics do not fit next to
            the actors on simple_spread N = 5 and 6: those raise MpeError before anything runs.
          - With MAPPO's shared recurrent actor (mpe_critic_gru_local, rIPPO): ONE tuple (base, gru, norm, v_out) (or
            [critic] * n) whose base reads obs_dim inputs, folded by rmappo_critic_params(critic, [obs_dim]) and run on
            every agent's observation record with that agent's own hidden state: critic_rnn_states and
            extras["final_critic_rnn_states"] are [n, N, 64], extras["critic_rnn_states"] [T, n, N, 64].
        Distinct per-agent recurrent local critics, local critics with the per-agent recurrent actors and local
        critics with any actor but MAPPO's raise NotImplementedError.  ValueError for centralized_critic=False without a
        critic, a shared critic on a program whose agents' obs_dims differ, a critic whose input width is not the
        agent's obs_dim, a critic whose activation, input LayerNorm or eps differ from the actors', or a
        critic_rnn_states other than a float32 [n, N, 64] tensor on the env's device.  Every refusal but MpeError
        happens before the world is bound; none changes the state or an epoch."""
        import torch
        world = self.world
        if action_mode not in ("softmax", "categorical"):
            raise ValueError("rollout_policy: action_mode must be 'softmax' or 'categorical', got %r" % (action_mode,))
        if record_log_probs and action_mode != "categorical":
            raise ValueError("rollout_policy: record_log_probs needs action_mode='categorical'")
        if not world.batched:
            raise ValueError("rollout_policy needs a batched env (make_env(..., num_envs=N))")
        if self._custom or self.discrete_action_input or self.force_discrete_action:
            raise NotImplementedError("rollout_policy: compiled scenarios with plain action vectors only")
        if len(policies) != self.n:
            raise ValueError("expected %d policies, got %d" % (self.n, len(policies)))
        if episode_length is not None and (int(episode_length) < 1 or int(n_steps) < int(episode_length)
                                           or int(n_steps) % int(episode_length) != 0):
            raise ValueError("rollout_policy: n_steps (%d) must be a positive multiple of episode_length (%d)"
                             % (int(n_steps), int(episode_length)))
        recurrent = any(_is_recurrent(p) for p in policies)
        recurrent_critic = critic is not None and _is_recurrent_critic(critic)
        if critic is not None:
            if recurrent_critic and not recurrent:
                raise NotImplementedError("rollout_policy: a recurrent critic (a tuple holding an nn.GRU) needs MAPPO's "
                                          "recurrent actor: rMAPPO pairs the actor's and the critic's recurrence")
            if recurrent and not recurrent_critic:
                raise NotImplementedError("rollout_policy: MAPPO's recurrent actor takes rMAPPO's recurrent critic "
                                          "(base, gru, norm, v_out): rMAPPO pairs the actor's and the critic's "
                                          "recurrence")
            if not recurrent and not any(_has_layer_norm(p) for p in policies):
                raise NotImplementedError("rollout_policy: critic needs MAPPO's MLP actor (LayerNorm layers); the "
                                          "two-hidden-layer and one-hidden-layer actors have no critic, and rMAPPO's "
                                          "critic is recurrent")
            if action_mode != "categorical":
                raise NotImplementedError("rollout_policy: critic needs action_mode='categorical'")
        local = None   # IPPO's local critics, folded and checked before the world is bound
        if not centralized_critic:
            if critic is None:
                raise ValueError("rollout_policy: centralized_critic=False selects IPPO's local critics and needs a "
                                 "critic")
            local = self._local_critic_fold(policies, critic, recurrent, critic_rnn_states)
        if (critic_rnn_states is not None or record_critic_rnn_states) and not recurrent_critic:
            raise ValueError("rollout_policy: critic_rnn_states and record_critic_rnn_states need rMAPPO's recurrent "
                             "critic (a critic tuple holding an nn.GRU)")
        if recurrent:
            if action_mode != "categorical":
                raise NotImplementedError("rollout_policy: MAPPO's recurrent actor has action_mode='categorical' only")
            if rnn_states is not None and episode_length is not None:
                raise ValueError("rollout_policy: rnn_states cannot be combined with episode_length (every episode "
                                 "starts from h = 0)")
            if critic_rnn_states is not None and episode_length is not None:
                raise ValueError("rollout_policy: critic_rnn_states cannot be combined with episode_length (every "
                                 "episode starts from h = 0)")
            sep = None   # rMAPPO's separated runner: distinct tuples on a program with per-agent recurrent actors
            if any(p is not policies[0] for p in policies) and self._has_gru_separated():
                sep = self._gru_separated_fold(policies, critic, rnn_states, critic_rnn_states)
            return self._rollout_policy_mlp(policies, n_steps, record_actions, per_step_rewards, record_observations,
                                            explore_seed, episode_length, True, record_log_probs, mappo=True,
                                            gru=(rnn_states, record_rnn_states, sep),
                                            rcritic=(critic, critic_rnn_states, record_critic_rnn_states)
                                            if critic is not None else None, local=local)
        if rnn_states is not None or record_rnn_states:
            raise ValueError("rollout_policy: rnn_states and record_rnn_states need MAPPO's recurrent actor "
                             "(a policy tuple with an nn.GRU)")
        if any(_has_layer_norm(p) for p in policies):
            if action_mode != "categorical":
                raise NotImplementedError("rollout_policy: MAPPO's actor (LayerNorm layers) has action_mode='categorical' "
                                          "only")
            if _mappo_hidden_widths(policies) - {MAPPO_HIDDEN}:
                raise NotImplementedError("rollout_policy: MAPPO's actor is built for hidden width %d only; got %s"
                                          % (MAPPO_HIDDEN, sorted(_mappo_hidden_widths(policies))))
            return self._rollout_policy_mlp(policies, n_steps, record_actions, per_step_rewards, record_observations,
                                            explore_seed, episode_length, True, record_log_probs, mappo=True,
                                            critic=critic, local=local)
        if any(_has_two_hidden_layers(p) for p in policies):
            return self._rollout_policy_mlp(policies, n_steps, record_actions, per_step_rewards, record_observations,
                                            explore_seed, episode_length, action_mode == "categorical", record_log_probs)
        if action_mode == "categorical":
            raise NotImplementedError("rollout_policy: action_mode='categorical' needs the two-hidden-layer actor "
                                      "(Linear -> ReLU -> Linear -> ReLU -> Linear)")
        if episode_length is not None:
            raise NotImplementedError("rollout_policy: episode_length needs the two-hidden-layer actor "
                                      "(Linear -> ReLU -> Linear -> ReLU -> Linear)")
        if record_observations or explore_seed is not None:
            raise NotImplementedError("rollout_policy: observation records and exploration need the two-hidden-layer "
                                      "actor (Linear -> ReLU -> Linear -> ReLU -> Linear)")
        nw = world.bind()
        N, T = nw.n_env, int(n_steps)
        keep, hidden = [], None
        ptrs = ([], [], [], [])
        for i, pol in enumerate(policies):
            if isinstance(pol, torch.nn.Module):
                lin = [m for m in pol.modules() if isinstance(m, torch.nn.Linear)]
                if len(lin) != 2:
                    raise ValueError("policy %d must be Linear -> ReLU -> Linear" % i)
                pol = (lin[0].weight, lin[0].bias, lin[1].weight, lin[1].bias)
            W1, b1, W2, b2 = [t.detach().to(device=nw.device, dtype=torch.float32) for t in pol]
            H = int(W1.shape[0])
            if hidden is None:
                hidden = H
            if H != hidden or tuple(W1.shape) != (H, nw.obs_dims[i]) or tuple(b1.shape) != (H,) or \
                    tuple(W2.shape) != (5, H) or tuple(b2.shape) != (5,):
                raise ValueError("policy %d: expected W1 [%d, %d], b1 [%d], W2 [5, %d], b2 [5]"
                                 % (i, hidden, nw.obs_dims[i], hidden, hidden))
            parts = (W1.t().contiguous(), b1.contiguous(), W2.contiguous(), b2.contiguous())   # W1 input-major for the kernel
            keep.append(parts)
            for lst, t in zip(ptrs, parts):
                lst.append(t.data_ptr())
        out = nw.out if self.reuse_buffers else nw.new_outputs()
        rew_steps = torch.empty((T, self.n, N), dtype=torch.float32, device=nw.device) if per_step_rewards else None
        actions = [torch.empty((T, N, 5), dtype=torch.float32, device=nw.device) for _ in range(self.n)] if record_actions else None
        nw.rollout_policy(*[_lib.ptr_array(p) for p in ptrs], hidden, T, out, self._flags(), rew_steps,
                          _lib.ptr_array([a.data_ptr() for a in actions]) if actions is not None else None)
        self._last_out = out
        world._obs_valid = False
        info_n = {'n': [{} for _ in range(self.n)]}
        return list(out.obs), list(out.rew_list), list(out.done_list), info_n, {"actions": actions, "rewards": rew_steps}

    def _has_gru_separated(self):
        """does the library have per-agent recurrent actors for this program?  (Asked without a device.)"""
        try:
            self.world.native_shapes().require_gru_separated()
        except _lib.MpeError:
            return False
        return True

    def _local_critic_fold(self, policies, critic, recurrent, critic_rnn_states):
        """IPPO's local critics, checked before the world is bound: the critic folded on one agent's obs_dim
        (mappo_actor_params on [obs_dim_k] per critic, or rmappo_critic_params(critic, [obs_dim]) for the recurrent
        one), its activation, input LayerNorm and eps against the actors', and critic_rnn_states [n, N, 64].  Returns
        (params, tanh, feature_norm, eps) as the centralized folds do."""
        import torch
        shapes = self.world.native_shapes()
        n, N, obs_dims = self.n, shapes.n_env, list(shapes.obs_dims)
        if recurrent:
            if any(p is not policies[0] for p in policies) and self._has_gru_separated():
                raise NotImplementedError("rollout_policy: local critics with per-agent recurrent actors (rMAPPO's "
                                          "separated runner) are not supported")
            if isinstance(critic, (tuple, list)) and len(critic) == n and all(_is_recurrent(c) for c in critic):
                if any(c is not critic[0] for c in critic):
                    raise NotImplementedError("rollout_policy: distinct per-agent recurrent local critics are not "
                                              "supported; pass one tuple ([critic] * n)")
                critic = critic[0]
            if len(set(obs_dims)) != 1:
                raise ValueError("rollout_policy: one shared local critic needs agents with equal obs_dims; got %s"
                                 % obs_dims)
            fold = rmappo_critic_params(critic, obs_dims[:1])
            actor = rmappo_actor_params(policies, obs_dims, list(shapes.act_dims))
        else:
            if isinstance(critic, torch.nn.Module):
                critics = [critic]
            elif isinstance(critic, (list, tuple)) and len(critic) in (1, n):
                critics = [critic[0]] if all(c is critic[0] for c in critic) else list(critic)
            else:
                raise ValueError("rollout_policy: the local critic must be one module, or a list of 1 or %d modules" % n)
            if len(critics) == 1 and len(set(obs_dims)) != 1:
                raise ValueError("rollout_policy: one shared local critic needs agents with equal obs_dims; got %s "
                                 "(pass %d per-agent critics)" % (obs_dims, n))
            dims = obs_dims[:1] if len(critics) == 1 else obs_dims
            try:
                fold = mappo_actor_params(critics, dims, [1] * len(critics))
            except ValueError as e:
                raise ValueError("rollout_policy: the local critic must be %s: %s" % (_LOCAL_CRITIC_SHAPE, e)) from None
            actor = mappo_actor_params(policies, obs_dims, list(shapes.act_dims))
        if fold[1:] != actor[1:]:
            raise ValueError("rollout_policy: the critic must use the actors' activation, input LayerNorm and eps (%s, "
                             "%s, %g); got (%s, %s, %g)" % ("Tanh" if actor[1] else "ReLU", actor[2], actor[3],
                                                           "Tanh" if fold[1] else "ReLU", fold[2], fold[3]))
        t = critic_rnn_states
        device = self._device()
        if t is not None and not (torch.is_tensor(t) and tuple(t.shape) == (n, N, MAPPO_HIDDEN)
                                  and t.dtype == torch.float32 and t.device == device):
            raise ValueError("rollout_policy: critic_rnn_states must be a float32 tensor %s on %s; got %s"
                             % ([n, N, MAPPO_HIDDEN], device, (tuple(t.shape), t.dtype, t.device)
                                if torch.is_tensor(t) else type(t).__name__))
        return fold

    def _device(self):
        """the env's device as bind() resolves it, without binding"""
        import torch
        world = self.world
        if world._native is not None:
            return world._native.device
        device = torch.device(world.device if world.device is not None else "cuda")
        if device.type == "cuda" and device.index is None and torch.cuda.is_available():
            device = torch.device("cuda", torch.cuda.current_device())
        return device

    def _gru_separated_fold(self, policies, critic, rnn_states, critic_rnn_states):
        """rMAPPO's separated runner, checked before the world is bound: every agent's actor folded by
        rmappo_actor_params on its own sizes, every agent's critic (a list of n recurrent tuples) by
        rmappo_critic_params, one activation, input LayerNorm and eps for all, and the two state tensors [n, N, 64].
        Returns (actor params per agent, (tanh, feature_norm, eps), critic params per agent or None)."""
        import torch
        shapes = self.world.native_shapes()
        n, N = self.n, shapes.n_env
        actors = []
        for i, pol in enumerate(policies):
            try:
                actors.append(rmappo_actor_params([pol], [shapes.obs_dims[i]], [shapes.act_dims[i]]))
            except ValueError as e:
                raise ValueError("rollout_policy: agent %d's recurrent actor: %s" % (i, e)) from None
        net = actors[0][1:]
        if any(a[1:] != net for a in actors):
            raise ValueError("rollout_policy: every agent's recurrent actor must use the same activation, input "
                             "LayerNorm and eps; got %s" % [("Tanh" if a[1] else "ReLU", a[2], a[3]) for a in actors])
        critics = None
        if critic is not None:
            if _is_recurrent(critic) or not (isinstance(critic, (list, tuple)) and len(critic) == n):
                raise ValueError("rollout_policy: per-agent recurrent actors take a list of %d recurrent critics, one "
                                 "per agent (rMAPPO's separated runner)" % n)
            critics = [rmappo_critic_params(c, shapes.obs_dims) for c in critic]
            if any(c[1:] != net for c in critics):
                raise ValueError("rollout_policy: every critic must use the actors' activation, input LayerNorm and "
                                 "eps (%s, %s, %g)" % ("Tanh" if net[0] else "ReLU", net[1], net[2]))
        device = self._device()
        for name, t in (("rnn_states", rnn_states), ("critic_rnn_states", critic_rnn_states)):
            if t is not None and not (torch.is_tensor(t) and tuple(t.shape) == (n, N, MAPPO_HIDDEN)
                                      and t.dtype == torch.float32 and t.device == device):
                raise ValueError("rollout_policy: %s must be a float32 tensor %s on %s; got %s"
                                 % (name, [n, N, MAPPO_HIDDEN], device, (tuple(t.shape), t.dtype, t.device)
                                    if torch.is_tensor(t) else type(t).__name__))
        return [a[0] for a in actors], net, (None if critics is None else [c[0] for c in critics])

    def compute_gae(self, rewards, values, final_values=None, gamma=0.99, gae_lambda=0.95, episode_length=None,
                    bootstrap=True, value_norm=None, normalize_advantages=False):
        """MAPPO's GAE advantages and returns (SharedReplayBuffer.compute_returns with use_gae) in one kernel launch
        (mpe_gae), plus PPO's advantage normalisation in a second one.  Any batched env, any source of values: the
        rollout_policy critics' extras or a trainer's own critic.

        rewards and values are float32 CUDA tensors [T, n, N] on the env's device (extras["rewards"] of
        per_step_rewards=True, extras["values"]); final_values is [n, N] (extras["final_values"]), or [E, n, N] with
        episode_length=L, E = T / L: episode e covers steps e*L .. e*L + L - 1 (rollout_policy's episode form); without
        episode_length the whole buffer is one episode.  value_norm (MAPPO's ValueNorm): None, or a float32 CUDA tensor
        (mean, std), [2] shared or [n, 2] one row per agent -- mean, var = value_normalizer.running_mean_var(); std =
        var.sqrt() -- and every value v is then denormalised as v * std + mean; it is read on the device, so the call
        never waits for the host and can be captured in a CUDA graph.  Per agent and world, t running backwards inside
        each episode:

            last   = t is the last step of its episode
            next   = last ? (bootstrap ? dv(final_values[e]) : 0) : dv[t + 1]
            carry  = last ? 0 : gae[t + 1]
            delta  = (r[t] + gamma * next) - dv[t]
            gae[t] = delta + (gamma * gae_lambda) * carry
            ret[t] = gae[t] + dv[t]

        in float32, every operation rounded in this order without fused multiply-adds (gamma and gae_lambda are rounded
        to float32 first, gamma * gae_lambda is one float32 product).  bootstrap=True treats an episode end as a
        time-limit truncation (continue with gamma * V of the final observation); bootstrap=False as terminal, MAPPO on
        MPE's behaviour, where final_values may be None.

        Returns (returns, advantages, stats): new float32 [T, n, N] tensors ret and gae.  The advantages are gae itself,
        not MAPPO's recomputed returns - dv; the two are equal in exact arithmetic and differ by at most the one float32
        rounding of ret.  normalize_advantages=True replaces them by (a - mean) / (std + 1e-5), mean and population std
        over all T * n * N entries, computed in float64 from per-block partial sums combined in a fixed order (two calls
        give the same bits), each entry float32((float64(a) - mean) / (std + 1e-5)); stats is then a float64 [2] tensor
        (mean, std), else None.  ValueError, before anything runs, for a non-batched env, tensors of the wrong shape,
        dtype, device or layout, a final_values that does not match episode_length, a value_norm that is not [2] or
        [n, 2], gamma or gae_lambda outside [0, 1], an episode_length that does not divide T, or bootstrap without
        final_values."""
        import torch
        world = self.world
        if not world.batched:
            raise ValueError("compute_gae needs a batched env (make_env(..., num_envs=N))")
        shapes = world.native_shapes()   # shapes first, the device (bind) once everything else is known to be valid
        n, N = shapes.n_agents, shapes.n_env

        def check_tensor(name, t, shape):
            if not torch.is_tensor(t) or t.dtype != torch.float32 or not t.is_contiguous():
                raise ValueError("compute_gae: %s must be a contiguous float32 tensor" % name)
            if tuple(t.shape) != tuple(shape):
                raise ValueError("compute_gae: %s must have shape %s, got %s" % (name, tuple(shape), tuple(t.shape)))

        if not torch.is_tensor(rewards) or rewards.dim() != 3 or rewards.shape[0] < 1:
            raise ValueError("compute_gae: rewards must be a [T, %d, %d] tensor with T >= 1" % (n, N))
        T = int(rewards.shape[0])
        check_tensor("rewards", rewards, (T, n, N))
        check_tensor("values", values, (T, n, N))
        if episode_length is not None and (int(episode_length) < 1 or T % int(episode_length) != 0):
            raise ValueError("compute_gae: episode_length (%s) must divide T (%d)" % (episode_length, T))
        for name, x in (("gamma", gamma), ("gae_lambda", gae_lambda)):
            if not 0.0 <= float(x) <= 1.0:   # also refuses NaN
                raise ValueError("compute_gae: %s must be a finite number in [0, 1], got %r" % (name, x))
        if bootstrap and final_values is None:
            raise ValueError("compute_gae: bootstrap=True needs final_values (bootstrap=False treats every episode "
                             "end as terminal)")
        if final_values is not None:
            check_tensor("final_values", final_values, (n, N) if episode_length is None
                         else (T // int(episode_length), n, N))
        per_agent = False
        if value_norm is not None:
            per_agent = torch.is_tensor(value_norm) and value_norm.dim() == 2
            check_tensor("value_norm", value_norm, (n, 2) if per_agent else (2,))
        # the env's device as bind() resolves it, so that wrong-device tensors are refused before the world is allocated
        device = self._device()
        for name, t in (("rewards", rewards), ("values", values), ("final_values", final_values),
                        ("value_norm", value_norm)):
            if t is not None and not (t.is_cuda and t.device == device):
                raise ValueError("compute_gae: %s must be a CUDA tensor on %s" % (name, device))
        nw = world.bind()
        flags = ((_lib.GAE_BOOTSTRAP if bootstrap else 0) | (_lib.GAE_NORMALIZE if normalize_advantages else 0) |
                 (_lib.GAE_PER_AGENT_VALUE_NORM if per_agent else 0))
        returns = torch.empty_like(rewards)
        advantages = torch.empty_like(rewards)
        ws = None
        if normalize_advantages:
            ws = torch.empty((nw.gae_workspace_bytes() + 7) // 8, dtype=torch.float64, device=nw.device)
        nw.gae(rewards, values, final_values if bootstrap else None, T, episode_length, gamma, gae_lambda, flags,
               value_norm, returns, advantages, ws)
        return returns, advantages, (ws[:2] if ws is not None else None)

    def _rollout_policy_mlp(self, policies, n_steps, record_actions, per_step_rewards, record_observations, explore_seed,
                            episode_length=None, categorical=False, record_log_probs=False, mappo=False, gru=None,
                            critic=None, rcritic=None, local=None):
        import torch
        world = self.world
        nw = world.bind()
        N, T = nw.n_env, int(n_steps)
        nw.require_mlp_actor()   # a program without the kernel is refused as such, before its heads are checked
        rnn = None
        if gru is not None:      # MAPPO's recurrent actor: gru = (rnn_states, record_rnn_states, separated fold)
            h0, record, sep = gru
            if sep is None:
                nw.require_gru_actor()
                params, tanh, feature_norm, eps = rmappo_actor_params(policies, nw.obs_dims, nw.act_dims)
                params = [params]    # one shared set
            else:                # every agent's own set (_gru_separated_fold)
                params, (tanh, feature_norm, eps), rparams = sep
            hidden = MAPPO_HIDDEN
            net = ((_lib.MAPPO_FEATURE_NORM if feature_norm else 0) | (_lib.MAPPO_TANH if tanh else 0), eps)
            shape = (self.n, N, MAPPO_HIDDEN)
            if h0 is not None:
                if not (torch.is_tensor(h0) and tuple(h0.shape) == shape and h0.dtype == torch.float32
                        and h0.device == torch.device(nw.device)):
                    raise ValueError("rollout_policy: rnn_states must be a float32 tensor %s on %s; got %s"
                                     % (list(shape), nw.device, (tuple(h0.shape), h0.dtype, h0.device)
                                        if torch.is_tensor(h0) else type(h0).__name__))
                h = h0.clone(memory_format=torch.contiguous_format)   # the kernel overwrites its state buffer
            elif episode_length is None:
                h = torch.zeros(shape, dtype=torch.float32, device=nw.device)
            else:                # every episode starts from h = 0 without reading the buffer
                h = torch.empty(shape, dtype=torch.float32, device=nw.device)
            rnn = (h, torch.empty((T,) + shape, dtype=torch.float32, device=nw.device) if record else None)
            if sep is not None:  # the workspace of the agents' fragment images
                rnn += (torch.empty(nw.gru_separated_workspace_bytes() // 4, dtype=torch.float32, device=nw.device),)
            if rcritic is not None:   # rMAPPO's recurrent critic: rcritic = (critic, critic_rnn_states, record)
                rmodule, ch0, crecord = rcritic
                if local is not None:   # rIPPO: checked by _local_critic_fold
                    rparams = local[0]
                    nw.require_critic_gru_local()
                elif sep is None:
                    rparams, ctanh, cfn, ceps = rmappo_critic_params(rmodule, nw.obs_dims)
                    if (ctanh, cfn, ceps) != (tanh, feature_norm, eps):
                        raise ValueError("rollout_policy: the critic must use the actor's activation, input LayerNorm "
                                         "and eps (%s, %s, %g); got (%s, %s, %g)"
                                         % ("Tanh" if tanh else "ReLU", feature_norm, eps, "Tanh" if ctanh else "ReLU",
                                            cfn, ceps))
                    nw.require_critic_gru()
                cshape = (N, MAPPO_HIDDEN) if sep is None and local is None else (self.n, N, MAPPO_HIDDEN)
                if ch0 is not None:
                    if not (torch.is_tensor(ch0) and tuple(ch0.shape) == cshape and ch0.dtype == torch.float32
                            and ch0.device == torch.device(nw.device)):
                        raise ValueError("rollout_policy: critic_rnn_states must be a float32 tensor %s on %s; got %s"
                                         % (list(cshape), nw.device, (tuple(ch0.shape), ch0.dtype, ch0.device)
                                            if torch.is_tensor(ch0) else type(ch0).__name__))
                    ch = ch0.clone(memory_format=torch.contiguous_format)   # the kernel overwrites its state buffer
                elif episode_length is None:
                    ch = torch.zeros(cshape, dtype=torch.float32, device=nw.device)
                else:            # every episode starts from h = 0 without reading the buffer
                    ch = torch.empty(cshape, dtype=torch.float32, device=nw.device)
                if sep is None:
                    rkeep = [t.to(device=nw.device, dtype=torch.float32).contiguous() for t in rparams]
                else:            # critic k's ten weights; the kernel takes one pointer array per weight
                    ckeep = [[t.to(device=nw.device, dtype=torch.float32).contiguous() for t in p] for p in rparams]
                    rkeep = [_lib.ptr_array([ckeep[k][j].data_ptr() for k in range(self.n)]) for j in range(10)]
                rcrit = (ch, torch.empty((T,) + cshape, dtype=torch.float32, device=nw.device) if crecord else None)
        elif mappo:
            params, tanh, feature_norm, eps = mappo_actor_params(policies, nw.obs_dims, nw.act_dims)
            hidden = MAPPO_HIDDEN
            net = ((_lib.MAPPO_FEATURE_NORM if feature_norm else 0) | (_lib.MAPPO_TANH if tanh else 0), eps)
            if local is not None:   # IPPO: checked by _local_critic_fold
                cparams = local[0]
                nw.require_local_critic(len(cparams))   # a program without the kernel, or critics that do not fit
            elif critic is not None:
                cparams, ctanh, cfn, ceps = mappo_critic_params(critic, nw.obs_dims)
                if (ctanh, cfn, ceps) != (tanh, feature_norm, eps):
                    raise ValueError("rollout_policy: the critic must use the actors' activation, input LayerNorm and "
                                     "eps (%s, %s, %g); got (%s, %s, %g)"
                                     % ("Tanh" if tanh else "ReLU", feature_norm, eps, "Tanh" if ctanh else "ReLU", cfn,
                                        ceps))
                nw.require_critic(len(cparams))   # a program without the kernel, or critics that do not fit
        else:
            params, hidden = mlp_actor_params(policies, nw.obs_dims, nw.act_dims)
            net = None
        keep = [[t.detach().to(device=nw.device, dtype=torch.float32).contiguous() for t in p] for p in params]
        if rnn is not None and len(rnn) == 2:
            w_ptrs = [t.data_ptr() for t in keep[0]]
        else:   # one pointer per agent for each weight
            w_ptrs = [_lib.ptr_array([keep[i][j].data_ptr() for i in range(self.n)]) for j in range(len(keep[0]))]
        out = nw.out if self.reuse_buffers else nw.new_outputs()
        dev = dict(dtype=torch.float32, device=nw.device)
        crit = None
        if critic is not None:
            ckeep = [[t.to(device=nw.device, dtype=torch.float32).contiguous() for t in p] for p in cparams]
            cw_ptrs = [_lib.ptr_array([ckeep[k][j].data_ptr() for k in range(len(ckeep))]) for j in range(6)]
            E = 1 if episode_length is None else T // int(episode_length)
            final_shape = (self.n, N) if episode_length is None else (E, self.n, N)
            crit = (len(ckeep), cw_ptrs, torch.empty((T, self.n, N), **dev), torch.empty(final_shape, **dev))
        rew_steps = torch.empty((T, self.n, N), **dev) if per_step_rewards else None
        if categorical:   # int32 [T, N, n_sub_i]: movement if movable, then utterance if it speaks
            n_sub = [int(bool(nw.desc.agent_movable[i])) + int(not nw.desc.agent_silent[i]) for i in range(self.n)]
            actions = [torch.empty((T, N, s), dtype=torch.int32, device=nw.device) for s in n_sub] if record_actions else None
        else:
            actions = [torch.empty((T, N, ad), **dev) for ad in nw.act_dims] if record_actions else None
        log_probs = torch.empty((T, self.n, N), **dev) if record_log_probs else None
        # the recurrent critic reads the rollout's observation records: scratch unless the caller asked for them
        need_obs = record_observations or rcritic is not None
        observations = [torch.empty((T, N, od), **dev) for od in nw.obs_dims] if need_obs else None
        seed = None if explore_seed is None else int(explore_seed) & 0xFFFFFFFFFFFFFFFF
        act_ptrs = _lib.ptr_array([a.data_ptr() for a in actions]) if actions is not None else None
        obs_ptrs = _lib.ptr_array([o.data_ptr() for o in observations]) if observations is not None else None
        extras = {"actions": actions, "rewards": rew_steps, "observations": observations if record_observations else None}
        if categorical:
            extras["log_probs"] = log_probs
        E, ep_rew, final = 1, None, None
        if episode_length is not None:
            E = T // int(episode_length)
            ep_rew = torch.empty((E, self.n, N), **dev)
            final = [torch.empty((E, N, od), **dev) for od in nw.obs_dims] if need_obs else None
        nw.rollout_policy_mlp(w_ptrs, hidden, T, out, self._flags(), episode_length=episode_length, categorical=categorical,
                              rew_steps=rew_steps, act_rec_ptrs=act_ptrs, obs_rec_ptrs=obs_ptrs,
                              final_obs_ptrs=_lib.ptr_array([o.data_ptr() for o in final]) if final is not None else None,
                              logp_steps=log_probs, ep_rew=ep_rew, explore_seed=seed, explore_epoch=self.explore_epoch,
                              mappo=net, gru=rnn, critic=crit, local_critic=local is not None)
        if rnn is not None:
            extras["final_rnn_states"], extras["rnn_states"] = rnn[:2]
        if rcritic is not None:   # on the same stream, after the rollout that wrote its input records
            values = torch.empty((T, self.n, N), **dev)
            final_values = torch.empty((self.n, N) if episode_length is None else (E, self.n, N), **dev)
            final_ptrs = out.obs_ptrs if final is None else _lib.ptr_array([o.data_ptr() for o in final])
            if sep is None:
                nw.critic_gru([t.data_ptr() for t in rkeep], obs_ptrs, final_ptrs, T, episode_length, rcrit[0],
                              rcrit[1], values, final_values, net, local=local is not None)
            else:
                nw.critic_gru_separated(rkeep, obs_ptrs, final_ptrs, T, episode_length, rcrit[0], rcrit[1], values,
                                        final_values, net)
            extras["values"], extras["final_values"] = values, final_values
            extras["final_critic_rnn_states"], extras["critic_rnn_states"] = rcrit
        if crit is not None:
            extras["values"], extras["final_values"] = crit[2], crit[3]
        if episode_length is None:
            reward_n = list(out.rew_list)
        else:
            reward_n = list(ep_rew.unbind(1))
            extras["final_observations"] = final if record_observations else None
        if seed is not None:
            self.explore_epoch += E
        self._last_out = out
        world._obs_valid = False
        info_n = {'n': [{} for _ in range(self.n)]}
        return list(out.obs), reward_n, list(out.done_list), info_n, extras

    # ---- user scenarios: native _set_action + World.step, callbacks in the user's torch code -------
    def _step_custom(self, action_n, nw, flags):
        import torch
        world = self.world
        acts = []
        for i, a in enumerate(action_n):
            if flags & _lib.FLAG_DISCRETE_ACTION_INPUT:      # already int32 [N, n_sub] on the device (_index_tensors)
                acts.append(a)
                continue
            t = a if torch.is_tensor(a) else torch.as_tensor(np.asarray(a, dtype=np.float32))
            t = t.to(device=nw.device, dtype=torch.float32).reshape(nw.n_env, self._act_dims[i]).contiguous()
            acts.append(t)
        nw.set_action(_lib.ptr_array([t.data_ptr() for t in acts]), flags)      # environment.py:87-88
        world.step()                                                            # :90
        obs_n = [self._get_obs(agent) for agent in self.agents]                 # :92-97
        reward_n = [torch.as_tensor(self._get_reward(agent), device=nw.device, dtype=torch.float32).expand(nw.n_env)
                    for agent in self.agents]
        if self.done_callback is None:
            done_n = [torch.zeros(nw.n_env, dtype=torch.bool, device=nw.device) for _ in self.agents]
        else:
            done_n = [self.done_callback(agent, world) for agent in self.agents]
        info_n = {'n': [self._get_info(agent) for agent in self.agents]}
        if self.shared_reward:                                                  # :100-102
            total = torch.stack(reward_n).sum(0)
            reward_n = [total] * self.n
        return obs_n, reward_n, done_n, info_n

    # ---- asynchronous stepping for host callers (batch extension) ------------------------------
    def step_async(self, action_n):
        """Enqueue H2D(actions) -> fused step -> D2H(outputs) on the current CUDA stream and return
        immediately; the caller overlaps its own host work (or another env's step) with the transfers and
        collects the results with `step_wait()`.  Host inputs only (NumPy / CPU tensors), batched mode."""
        world = self.world
        if not world.batched:
            raise ValueError("step_async needs a batched env (make_env(..., num_envs=N))")
        if getattr(self, "_pending", None) is not None:
            raise RuntimeError("step_async called twice without step_wait")
        if self._custom:
            raise NotImplementedError("step_async is not available for user scenarios (TorchScenario): their "
                                      "observation / reward callbacks run as torch ops after the native step")
        if self.discrete_action_input:
            raise NotImplementedError("step_async takes action vectors; integer actions go through step()")
        if len(action_n) != self.n:
            raise ValueError("expected %d actions, got %d" % (self.n, len(action_n)))
        nw = world.bind()
        self.agents = world.policy_agents
        mode, payload = self._classify(action_n, nw)
        if mode == "cuda":
            raise ValueError("step_async is for host buffers; CUDA-tensor steps are already asynchronous")
        hs = nw.host_staging()
        ptrs = []
        for i, a in enumerate(payload):
            if mode == "pinned":
                ptrs.append(a.data_ptr())
            else:
                hs["host_act"][i].copy_(a)
                ptrs.append(hs["host_act"][i].data_ptr())
        hout = nw.step_host(_lib.ptr_array(ptrs), self._flags(), with_info=self._native_info)
        ev = nw.torch.cuda.Event()
        ev.record(nw.torch.cuda.current_stream(nw.device))
        self._pending = (hout, ev, payload, not hasattr(action_n[0], "dim"))
        world._obs_valid = False

    def step_wait(self):
        """Block until the step enqueued by `step_async` has landed in host memory; returns what `step` returns."""
        if getattr(self, "_pending", None) is None:
            raise RuntimeError("step_wait without step_async")
        hout, ev, _keepalive, as_numpy = self._pending
        self._pending = None
        ev.synchronize()
        self._last_out = hout
        return self._pack_batched(self.world.bind(), hout, as_numpy=as_numpy)

    # ---- input classification ---------------------------------------------------------------
    def _to_cpu_tensor(self, a, i):
        import torch
        t = torch.as_tensor(np.ascontiguousarray(np.asarray(a, dtype=np.float32)))
        return t.reshape(self.world.batch_size, self._act_dims[i])

    def _classify(self, action_n, nw):
        import torch
        N = self.world.batch_size
        if all(torch.is_tensor(a) and a.is_cuda for a in action_n):
            payload = []
            for i, a in enumerate(action_n):
                if a.device != nw.device:
                    raise ValueError("action_n[%d] lives on %s but this env's worlds live on %s" % (i, a.device, nw.device))
                if a.shape != (N, self._act_dims[i]):
                    raise ValueError("action_n[%d] must have shape (%d, %d), got %s" %
                                     (i, N, self._act_dims[i], tuple(a.shape)))
                if a.dtype != torch.float32 or not a.is_contiguous() or a.data_ptr() % 16:
                    a = a.to(torch.float32).contiguous().clone()
                payload.append(a)
            return "cuda", payload
        payload = []
        pinned = True
        for i, a in enumerate(action_n):
            if torch.is_tensor(a):
                a = a.detach()
                if a.is_cuda:
                    a = a.cpu()
                a = a.reshape(N, -1)
                ok = a.dtype == torch.float32 and a.is_contiguous() and a.is_pinned()
                if not ok:
                    a = a.to(torch.float32).contiguous()
                pinned = pinned and ok
            else:
                a = self._to_cpu_tensor(a, i)
                pinned = False
            if a.shape != (N, self._act_dims[i]):
                raise ValueError("action_n[%d] must have %d x %d elements, got shape %s" %
                                 (i, N, self._act_dims[i], tuple(a.shape)))
            payload.append(a)
        return ("pinned" if pinned else "host"), payload

    # ---- output packing -----------------------------------------------------------------------
    def _info_list(self, nw, out, batched):
        if self.info_callback is None:
            return [{} for _ in range(self.n)]
        if self._native_info:
            return [nw.benchmark_data(i, batched, out) for i in range(self.n)]
        return [self.info_callback(agent, self.world) for agent in self.agents]

    def _pack_batched(self, nw, out, as_numpy=False):
        obs_n = list(out.obs)
        reward_n = list(out.rew_list)
        done_n = list(out.done_list)
        if self.done_callback is not None:
            done_n = [self.done_callback(agent, self.world) for agent in self.agents]
        info_n = {'n': self._info_list(nw, out, True)}
        if out.slab.device.type == "cpu" and not self.reuse_buffers:
            # pinned staging slabs are reused every other step: the caller gets its own copies (the reference
            # returns freshly allocated arrays, and trainers keep them in replay buffers by reference)
            own = lambda t: t.clone() if hasattr(t, "clone") else t
            obs_n, reward_n, done_n = [own(o) for o in obs_n], [own(r) for r in reward_n], [own(d) for d in done_n]
            info_n = {'n': [tuple(own(x) for x in e) if isinstance(e, tuple) else own(e) for e in info_n['n']]}
        if as_numpy:
            obs_n = [o.numpy() for o in obs_n]
            reward_n = [r.numpy() for r in reward_n]
            done_n = [d.numpy() if hasattr(d, "numpy") else d for d in done_n]
        return obs_n, reward_n, done_n, info_n

    def _pack_scalar(self, nw, hout):
        if getattr(hout, "obs_np", None) is not None:       # pinned host outputs: plain NumPy views
            obs_n = [o[0].astype(np.float64) for o in hout.obs_np]
            rew = hout.rew_np[:, 0].astype(np.float64)
            done_n = [bool(d) for d in hout.done_np[:, 0]]
        else:
            obs_n = [o[0].detach().to("cpu").numpy().astype(np.float64) for o in hout.obs]
            rew = hout.rew[:, 0].detach().to("cpu").numpy().astype(np.float64)
            done_n = [bool(d) for d in hout.done[:, 0].detach().to("cpu")]
        reward_n = [rew[i] for i in range(self.n)]
        if self.done_callback is not None:
            done_n = [self.done_callback(agent, self.world) for agent in self.agents]
        info_n = {'n': self._info_list(nw, hout, False)}
        return obs_n, reward_n, done_n, info_n

    # ------------------------------------------------------------------------------------------
    def reset(self, mask=None, seed=None):
        """environment.py:106-116.  `mask` ([N] bool) resets a subset of the worlds (batched
        extension); observations are returned for every world."""
        world = self.world
        nw = world.bind()
        if mask is None and seed is None:
            self.reset_callback(world)
        else:
            self.reset_callback(world, mask=mask, seed=seed)
        self._reset_render()
        self.agents = world.policy_agents
        if self._custom:
            return [self._get_obs(agent) for agent in self.agents]
        out = nw.out if (self.reuse_buffers or not world.batched) else nw.new_outputs()
        nw.observe(out, 0, with_info=False)
        world._obs_valid = False
        if world.batched:
            return list(out.obs)
        return [o[0].detach().to("cpu").numpy().astype(np.float64) for o in out.obs]

    # ---- per-agent accessors kept for API compatibility (environment.py:119-141) --------------
    def _get_info(self, agent):
        if self.info_callback is None:
            return {}
        return self.info_callback(agent, self.world)

    def _get_obs(self, agent):
        if self.observation_callback is None:
            return np.zeros(0)
        return self.observation_callback(agent, self.world)

    def _get_done(self, agent):
        if self.done_callback is None:
            return False
        return self.done_callback(agent, self.world)

    def _get_reward(self, agent):
        if self.reward_callback is None:
            return 0.0
        return self.reward_callback(agent, self.world)

    def _set_action(self, action, agent, action_space, time=None):
        """environment.py:144-192 for ONE agent: decodes into agent.action.u / .c via the native
        set_action kernel (all agents are decoded; the other agents' inputs are zero)."""
        import torch
        nw = self.world.bind()
        idx = self.world._agent_index(agent)
        acts = [torch.zeros(nw.n_env, ad, device=nw.device) for ad in self._act_dims]
        acts[idx] = torch.as_tensor(np.asarray(action, dtype=np.float32) if not torch.is_tensor(action) else action,
                                    dtype=torch.float32, device=nw.device).reshape(nw.n_env, -1).contiguous()
        keep_u, keep_c = nw.act_u.clone(), nw.act_c.clone()
        nw.set_action(_lib.ptr_array([t.data_ptr() for t in acts]), self._flags())
        s = nw.speaker_slot(idx)
        new_u = nw.act_u[idx].clone()
        new_c = nw.act_c[s * nw.dim_c:(s + 1) * nw.dim_c].clone() if s >= 0 else None
        nw.act_u.copy_(keep_u)
        nw.act_c.copy_(keep_c)
        nw.act_u[idx] = new_u
        if new_c is not None:
            nw.act_c[s * nw.dim_c:(s + 1) * nw.dim_c] = new_c

    # ---- rendering: a headless rasteriser stands in for the pyglet viewer (SURVEY.md 8(f) rank 4) ---
    def _reset_render(self):
        self.render_geoms = None
        self.render_geoms_xform = None

    def render(self, mode='human', world_index=0):
        """environment.py:200-263 without a window: returns one uint8 [700, 700, 3] image per viewer
        (one shared viewer, or one per agent when shared_viewer=False) of world `world_index`;
        mode 'human' additionally prints the communication line the reference prints (:201-213)."""
        from .raster import draw_world
        world = self.world
        nw = world.bind()
        pv = nw.agent_pv[:, world_index].detach().to("cpu").numpy().astype(np.float64)
        lm = nw.lm_p[:, world_index].detach().to("cpu").numpy().astype(np.float64)[:len(world.landmarks)]
        if mode == 'human':
            alphabet = 'ABCDEFGHIJKLMNOPQRSTUVWXYZ'
            message = ''
            for agent in world.agents:
                for i, other in enumerate(world.agents):
                    if other is agent:
                        continue
                    s = nw.speaker_slot(i)
                    c = np.zeros(0) if s < 0 else nw.comm[s * nw.dim_c:(s + 1) * nw.dim_c, world_index].detach().to("cpu").numpy()
                    word = '_' if (c.size == 0 or np.all(c == 0)) else alphabet[int(np.argmax(c))]
                    message += (other.name + ' to ' + agent.name + ': ' + word + '   ')
            print(message)
        ents = world.entities
        pos = np.concatenate([pv[:, 0:2], lm], axis=0) if len(lm) else pv[:, 0:2]
        sizes = [e.size for e in ents]
        colors = [e.color for e in ents]
        alphas = [0.5 if 'agent' in e.name else 1.0 for e in ents]
        results = []
        for i in range(len(self.viewers)):
            center = (0.0, 0.0) if self.shared_viewer else tuple(pv[i, 0:2])
            results.append(draw_world(pos, sizes, colors, alphas, center=center))
        return results


# ---- the two-hidden-layer actor of rollout_policy (MADDPG's mlp_model) ------------------------------
_MLP_SHAPE = ("nn.Sequential(Linear(obs_dim, H), ReLU(), Linear(H, H), ReLU(), Linear(H, act_dim)) or a tuple "
              "(W1, b1, W2, b2, W3, b3)")


def _has_two_hidden_layers(pol):
    """does this policy ask for the two-hidden-layer actor?  (A 6-tuple, or a module with three Linear layers; whether
    the module really is Linear -> ReLU -> Linear -> ReLU -> Linear is checked by mlp_actor_params.)"""
    import torch
    if isinstance(pol, torch.nn.Module):
        return sum(isinstance(m, torch.nn.Linear) for m in pol.modules()) == 3
    return isinstance(pol, (tuple, list)) and len(pol) == 6


def mlp_actor_params(policies, obs_dims, act_dims=None):
    """policies -> ([(W1, b1, W2, b2, W3, b3) per agent], H) in torch's Linear layout, or ValueError.  A module must be
    an nn.Sequential whose layers are exactly Linear, ReLU, Linear, ReLU, Linear (types and order are checked: that
    order is the one the kernel evaluates); shapes must be W1 [H, obs_dim_i], b1 [H], W2 [H, H], b2 [H],
    W3 [act_dim_i, H], b3 [act_dim_i] with one H for all agents.  act_dims None means 5 (movement only) for every agent.
    No device is needed."""
    import torch
    if act_dims is None:
        act_dims = [5] * len(obs_dims)
    if len(policies) != len(obs_dims):
        raise ValueError("expected %d policies, got %d" % (len(obs_dims), len(policies)))
    params, hidden = [], None
    for i, pol in enumerate(policies):
        if isinstance(pol, torch.nn.Module):
            layers = [m for m in pol.modules() if not list(m.children())]
            names = " -> ".join(type(m).__name__ for m in layers)
            ok = (isinstance(pol, torch.nn.Sequential) and len(layers) == 5
                  and all(isinstance(layers[k], torch.nn.Linear) for k in (0, 2, 4))
                  and all(type(layers[k]) is torch.nn.ReLU for k in (1, 3)))
            if not ok:
                raise ValueError("policy %d must be %s; got %s (%s)" % (i, _MLP_SHAPE, type(pol).__name__, names))
            if any(layers[k].bias is None for k in (0, 2, 4)):
                raise ValueError("policy %d: every Linear layer needs a bias" % i)
            pol = (layers[0].weight, layers[0].bias, layers[2].weight, layers[2].bias, layers[4].weight, layers[4].bias)
        elif not (isinstance(pol, (tuple, list)) and len(pol) == 6):
            raise ValueError("policy %d must be %s" % (i, _MLP_SHAPE))
        ts = [t if torch.is_tensor(t) else torch.as_tensor(np.asarray(t, dtype=np.float32)) for t in pol]
        if ts[0].dim() != 2:
            raise ValueError("policy %d: W1 must be a matrix [H, %d], got shape %s" % (i, obs_dims[i], tuple(ts[0].shape)))
        H = int(ts[0].shape[0])
        if hidden is None:
            hidden = H
        ad = act_dims[i]
        want = ((hidden, obs_dims[i]), (hidden,), (hidden, hidden), (hidden,), (ad, hidden), (ad,))
        got = tuple(tuple(t.shape) for t in ts)
        if got != want:
            raise ValueError("policy %d: expected W1 [%d, %d], b1 [%d], W2 [%d, %d], b2 [%d], W3 [%d, %d], b3 [%d]; got %s"
                             % (i, hidden, obs_dims[i], hidden, hidden, hidden, hidden, ad, hidden, ad,
                                ", ".join(str(list(s)) for s in got)))
        params.append(tuple(ts))
    return params, hidden


# ---- MAPPO's MLP actor (MLPBase with layer_N = 1 and a categorical ACTLayer head) ----------------------------------
MAPPO_HIDDEN = 64
_MAPPO_SHAPE = ("nn.Sequential([LayerNorm(obs_dim)], Linear(obs_dim, 64), Act, LayerNorm(64), Linear(64, 64), Act, "
                "LayerNorm(64), Linear(64, act_dim)) with Act = ReLU() or Tanh()")


def _has_layer_norm(pol):
    """does this policy ask for MAPPO's actor?  (A module with a LayerNorm; mappo_actor_params checks the rest.)"""
    import torch
    return isinstance(pol, torch.nn.Module) and any(isinstance(m, torch.nn.LayerNorm) for m in pol.modules())


def _mappo_hidden_widths(policies):
    """the output width of every MAPPO policy's first Linear layer (what the kernel's H would be)"""
    import torch
    out = set()
    for pol in policies:
        lin = [m for m in pol.modules() if isinstance(m, torch.nn.Linear)] if isinstance(pol, torch.nn.Module) else []
        if lin:
            out.add(int(lin[0].out_features))
    return out


def mappo_actor_params(policies, obs_dims, act_dims=None):
    """MAPPO's actor -> (params, tanh, feature_norm, eps), or ValueError.  Every policy must be an nn.Sequential whose
    layers are exactly
        [LayerNorm(obs_dim_i)], Linear(obs_dim_i, 64), Act, LayerNorm(64), Linear(64, 64), Act, LayerNorm(64),
        Linear(64, act_dim_i)
    with Act = ReLU() or Tanh(), the same in both places and for all agents; the input LayerNorm (MAPPO's
    use_feature_normalization) for all agents or none; every LayerNorm with elementwise_affine=True and one eps for all;
    every Linear with a bias.  One module object may serve several agents (MAPPO's share_policy).  act_dims None means 5
    for every agent.

    params[i] = (W1', b1', W2', b2', W3', b3') in float64, torch's Linear layout: the network with each LayerNorm's
    affine folded into the Linear after it, W' = W diag(gamma), b' = b + W beta, so that the kernel needs only the
    parameter-free (x - mu) * rsqrt(var + eps).  No device is needed."""
    import torch
    nn = torch.nn
    if act_dims is None:
        act_dims = [5] * len(obs_dims)
    if len(policies) != len(obs_dims):
        raise ValueError("expected %d policies, got %d" % (len(obs_dims), len(policies)))
    H = MAPPO_HIDDEN
    params, acts, feature_norms, eps = [], set(), set(), set()
    for i, pol in enumerate(policies):
        layers = [m for m in pol.modules() if not list(m.children())] if isinstance(pol, nn.Module) else []
        names = " -> ".join(type(m).__name__ for m in layers)
        fn = len(layers) == 8 and type(layers[0]) is nn.LayerNorm
        body = layers[1:] if fn else layers
        ok = (isinstance(pol, nn.Sequential) and len(body) == 7
              and all(type(body[k]) is nn.Linear for k in (0, 3, 6))
              and all(type(body[k]) is nn.LayerNorm for k in (2, 5))
              and type(body[1]) in (nn.ReLU, nn.Tanh) and type(body[4]) is type(body[1]))
        if not ok:
            raise ValueError("policy %d must be %s; got %s (%s)" % (i, _MAPPO_SHAPE, type(pol).__name__, names))
        lins, norms = (body[0], body[3], body[6]), ((layers[0] if fn else None), body[2], body[5])
        if any(ln is not None and ln.weight is None for ln in norms):
            raise ValueError("policy %d: every LayerNorm needs elementwise_affine=True" % i)
        if any(lin.bias is None for lin in lins):
            raise ValueError("policy %d: every Linear layer needs a bias" % i)
        od, ad = obs_dims[i], act_dims[i]
        want = ((H, od), (H, H), (ad, H))
        got = tuple(tuple(lin.weight.shape) for lin in lins)
        ln_want = ((od,), (H,), (H,))
        ln_got = tuple(None if ln is None else tuple(ln.normalized_shape) for ln in norms)
        if got != want or any(g is not None and g != w for g, w in zip(ln_got, ln_want)):
            raise ValueError("policy %d: expected Linear weights %s and LayerNorm shapes %s (hidden width %d only); got "
                             "%s and %s" % (i, list(want), list(ln_want), H, list(got), list(ln_got)))
        acts.add(type(body[1]))
        feature_norms.add(fn)
        eps.update(float(ln.eps) for ln in norms if ln is not None)
        p = []
        for lin, ln in zip(lins, norms):
            W, b = lin.weight.detach().to(torch.float64), lin.bias.detach().to(torch.float64)
            if ln is not None:
                g = ln.weight.detach().to(torch.float64)
                beta = ln.bias.detach().to(torch.float64) if ln.bias is not None else torch.zeros_like(g)
                W, b = W * g, b + W @ beta
            p += [W, b]
        params.append(tuple(p))
    if len(acts) != 1:
        raise ValueError("every policy must use the same activation (ReLU or Tanh); got %s"
                         % sorted(a.__name__ for a in acts))
    if len(feature_norms) != 1:
        raise ValueError("the input LayerNorm (feature normalisation) must be on for every policy or for none")
    if len(eps) != 1:
        raise ValueError("every LayerNorm must have the same eps; got %s" % sorted(eps))
    return params, acts.pop() is nn.Tanh, feature_norms.pop(), eps.pop()


# ---- MAPPO's centralized critic (R_Critic with use_centralized_V, non-recurrent) -------------------------------------
_CRITIC_SHAPE = ("nn.Sequential([LayerNorm(D)], Linear(D, 64), Act, LayerNorm(64), Linear(64, 64), Act, LayerNorm(64), "
                 "Linear(64, 1)) with Act = ReLU() or Tanh() and D the sum of the agents' observation sizes")

_LOCAL_CRITIC_SHAPE = ("nn.Sequential([LayerNorm(D)], Linear(D, 64), Act, LayerNorm(64), Linear(64, 64), Act, "
                       "LayerNorm(64), Linear(64, 1)) with Act = ReLU() or Tanh() and D the agent's observation size")


def mappo_critic_params(critic, obs_dims):
    """MAPPO's centralized critic -> (params, tanh, feature_norm, eps), or ValueError.  critic is one module (a shared
    critic), a list of one, or a list of len(obs_dims) modules; a list whose entries are all the same object is one
    shared critic ([critic] * n, MAPPO's share_policy), any other list of len(obs_dims) per-agent critics.  Each must be
        [LayerNorm(D)], Linear(D, 64), Act, LayerNorm(64), Linear(64, 64), Act, LayerNorm(64), Linear(64, 1)
    (D = sum(obs_dims), the width of share_obs) under the rules of mappo_actor_params, with one activation, input
    LayerNorm and eps for all.  params: one (W1', b1', W2', b2', W3', b3') per critic in float64, each LayerNorm's
    affine folded into the Linear after it as mappo_actor_params folds the actor's.  No device is needed."""
    import torch
    n, D = len(obs_dims), int(sum(obs_dims))
    if isinstance(critic, torch.nn.Module):
        critics = [critic]
    elif isinstance(critic, (list, tuple)) and len(critic) in (1, n):
        critics = [critic[0]] if all(c is critic[0] for c in critic) else list(critic)
    else:
        raise ValueError("critic must be one module, or a list of 1 or %d modules; got %s"
                         % (n, "a list of %d" % len(critic) if isinstance(critic, (list, tuple))
                            else type(critic).__name__))
    try:
        return mappo_actor_params(critics, [D] * len(critics), [1] * len(critics))
    except ValueError as e:
        raise ValueError("critic must be %s: %s" % (_CRITIC_SHAPE, e)) from None


# ---- MAPPO's recurrent actor (R_Actor with use_recurrent_policy, recurrent_N = 1, share_policy) -----------------------
_RMAPPO_SHAPE = ("(base, gru, norm, head) with base = nn.Sequential([LayerNorm(obs_dim)], Linear(obs_dim, 64), Act, "
                 "LayerNorm(64), Linear(64, 64), Act, LayerNorm(64)), Act = ReLU() or Tanh(), gru = nn.GRU(64, 64), "
                 "norm = LayerNorm(64), head = Linear(64, act_dim)")


def _is_recurrent(pol):
    """does this policy ask for MAPPO's recurrent actor?  (A tuple holding an nn.GRU; rmappo_actor_params checks it.)"""
    import torch
    return isinstance(pol, (tuple, list)) and any(isinstance(m, torch.nn.GRU) for m in pol)


def _is_recurrent_critic(critic):
    """does this critic ask for rMAPPO's recurrent critic?  (A tuple holding an nn.GRU, or a list of such tuples;
    rmappo_critic_params checks the rest.)"""
    return _is_recurrent(critic) or (isinstance(critic, (tuple, list)) and len(critic) > 0
                                     and all(_is_recurrent(c) for c in critic))


def _fold_layer_norm(W, b, ln):
    """W, b of the Linear (or GRU input map) after LayerNorm ln, in float64, with ln's affine folded in:
    W' = W diag(gamma), b' = b + W beta"""
    import torch
    W, b = W.detach().to(torch.float64), b.detach().to(torch.float64)
    if ln is None:
        return W, b
    g = ln.weight.detach().to(torch.float64)
    beta = ln.bias.detach().to(torch.float64) if ln.bias is not None else torch.zeros_like(g)
    return W * g, b + W @ beta


def rmappo_actor_params(policies, obs_dims, act_dims=None):
    """MAPPO's recurrent actor -> (params, tanh, feature_norm, eps), or ValueError.  policies must be one 4-tuple
    (base, gru, norm, head) shared by every agent ([actor] * n, MAPPO's share_policy; distinct tuples raise
    NotImplementedError even when their values are equal):
        base = nn.Sequential([LayerNorm(obs_dim)], Linear(obs_dim, 64), Act, LayerNorm(64), Linear(64, 64), Act,
               LayerNorm(64))   -- MAPPO's MLPBase, Act = ReLU() or Tanh() in both places
        gru  = nn.GRU(64, 64) with num_layers=1, bias=True, bidirectional=False
        norm = nn.LayerNorm(64), head = nn.Linear(64, act_dim)
    Every LayerNorm affine with one eps, every Linear with a bias, and every agent with the same obs_dim and act_dim
    (act_dims None means 5).  From an on-policy R_Actor `a`: (nn.Sequential(a.base.feature_norm, *a.base.mlp.fc1,
    *a.base.mlp.fc2[0]), a.rnn.rnn, a.rnn.norm, a.act.action_out.linear).

    params = (W1, b1, W2, b2, W_ih, b_ih, W_hh, b_hh, W3, b3) in float64, torch's layouts, with each LayerNorm's affine
    folded into what follows it (the base's last one into W_ih, b_ih; norm into the head), so that the kernel needs only
    the parameter-free (x - mu) * rsqrt(var + eps).  No device is needed."""
    import torch
    nn = torch.nn
    if act_dims is None:
        act_dims = [5] * len(obs_dims)
    if len(policies) != len(obs_dims):
        raise ValueError("expected %d policies, got %d" % (len(obs_dims), len(policies)))
    pol = policies[0]
    if any(p is not pol for p in policies):
        raise NotImplementedError("the recurrent actor must be one policy object shared by every agent ([actor] * n, "
                                  "MAPPO's share_policy); distinct per-agent recurrent policies are not supported")
    if len(set(obs_dims)) != 1 or len(set(act_dims)) != 1:
        raise ValueError("one shared policy needs every agent to have the same observation and action sizes; got %s "
                         "and %s" % (list(obs_dims), list(act_dims)))
    if not (isinstance(pol, (tuple, list)) and len(pol) == 4):
        raise ValueError("the recurrent actor must be %s" % _RMAPPO_SHAPE)
    base, gru, norm, head = pol
    H, od, ad = MAPPO_HIDDEN, obs_dims[0], act_dims[0]
    layers = [m for m in base.modules() if not list(m.children())] if isinstance(base, nn.Module) else []
    fn = len(layers) == 7 and type(layers[0]) is nn.LayerNorm
    body = layers[1:] if fn else layers
    if not (isinstance(base, nn.Sequential) and len(body) == 6 and type(body[0]) is nn.Linear
            and type(body[3]) is nn.Linear and type(body[2]) is nn.LayerNorm and type(body[5]) is nn.LayerNorm
            and type(body[1]) in (nn.ReLU, nn.Tanh) and type(body[4]) is type(body[1])):
        raise ValueError("the recurrent actor's base must be %s; got %s (%s)"
                         % (_RMAPPO_SHAPE, type(base).__name__, " -> ".join(type(m).__name__ for m in layers)))
    if type(gru) is not nn.GRU:
        raise ValueError("the recurrent actor's second part must be an nn.GRU; got %s" % type(gru).__name__)
    if gru.num_layers != 1 or gru.bidirectional or not gru.bias or gru.input_size != H or gru.hidden_size != H:
        raise ValueError("the recurrent actor's GRU must be nn.GRU(%d, %d) with num_layers=1, bias=True and "
                         "bidirectional=False; got %r" % (H, H, gru))
    if type(norm) is not nn.LayerNorm or tuple(norm.normalized_shape) != (H,):
        raise ValueError("the recurrent actor's third part must be nn.LayerNorm(%d); got %r" % (H, norm))
    if type(head) is not nn.Linear or tuple(head.weight.shape) != (ad, H):
        raise ValueError("the recurrent actor's head must be nn.Linear(%d, %d); got %r" % (H, ad, head))
    norms = ((layers[0] if fn else None), body[2], body[5], norm)
    if any(ln is not None and ln.weight is None for ln in norms):
        raise ValueError("the recurrent actor: every LayerNorm needs elementwise_affine=True")
    if any(lin.bias is None for lin in (body[0], body[3], head)):
        raise ValueError("the recurrent actor: every Linear layer needs a bias")
    got = (tuple(body[0].weight.shape), tuple(body[3].weight.shape))
    ln_got = tuple(None if ln is None else tuple(ln.normalized_shape) for ln in norms[:3])
    if got != ((H, od), (H, H)) or any(g is not None and g != w for g, w in zip(ln_got, ((od,), (H,), (H,)))):
        raise ValueError("the recurrent actor's base: expected Linear weights %s and LayerNorm shapes %s; got %s and %s"
                         % ([(H, od), (H, H)], [(od,), (H,), (H,)], list(got), list(ln_got)))
    eps = {float(ln.eps) for ln in norms if ln is not None}
    if len(eps) != 1:
        raise ValueError("every LayerNorm must have the same eps; got %s" % sorted(eps))
    W1, b1 = _fold_layer_norm(body[0].weight, body[0].bias, norms[0])
    W2, b2 = _fold_layer_norm(body[3].weight, body[3].bias, body[2])
    W_ih, b_ih = _fold_layer_norm(gru.weight_ih_l0, gru.bias_ih_l0, body[5])
    W_hh, b_hh = _fold_layer_norm(gru.weight_hh_l0, gru.bias_hh_l0, None)
    W3, b3 = _fold_layer_norm(head.weight, head.bias, norm)
    return (W1, b1, W2, b2, W_ih, b_ih, W_hh, b_hh, W3, b3), type(body[1]) is nn.Tanh, fn, eps.pop()


# ---- rMAPPO's recurrent centralized critic (R_Critic with use_recurrent_policy, recurrent_N = 1, use_centralized_V) ----
_RCRITIC_SHAPE = ("(base, gru, norm, v_out) with base = nn.Sequential([LayerNorm(D)], Linear(D, 64), Act, LayerNorm(64), "
                  "Linear(64, 64), Act, LayerNorm(64)), Act = ReLU() or Tanh(), gru = nn.GRU(64, 64), norm = "
                  "LayerNorm(64), v_out = Linear(64, 1) and D the sum of the agents' observation sizes")


def rmappo_critic_params(critic, obs_dims):
    """rMAPPO's recurrent centralized critic -> (params, tanh, feature_norm, eps), or ValueError.  critic is one tuple
    (base, gru, norm, v_out), or a list of 1 or len(obs_dims) entries that are all that same tuple object ([critic] * n,
    a shared critic); distinct tuples raise NotImplementedError.  The tuple is checked under the rules of
    rmappo_actor_params with input width D = sum(obs_dims) (share_obs) and head Linear(64, 1).  From an on-policy
    R_Critic `c`: (nn.Sequential(c.base.feature_norm, *c.base.mlp.fc1, *c.base.mlp.fc2[0]), c.rnn.rnn, c.rnn.norm,
    c.v_out).  params = (W1, b1, W2, b2, W_ih, b_ih, W_hh, b_hh, W3, b3) in float64, folded as rmappo_actor_params
    folds the actor (W1 [64, D], W3 [1, 64], b3 [1]).  No device is needed."""
    n, D = len(obs_dims), int(sum(obs_dims))
    if _is_recurrent(critic):
        one = critic
    elif isinstance(critic, (tuple, list)) and len(critic) in (1, n) and all(_is_recurrent(c) for c in critic):
        if any(c is not critic[0] for c in critic):
            raise NotImplementedError("the recurrent critic must be one tuple shared by every agent ([critic] * n); "
                                      "distinct per-agent recurrent critics are not supported")
        one = critic[0]
    else:
        raise ValueError("the recurrent critic must be one tuple %s, or a list of 1 or %d of that same tuple"
                         % (_RCRITIC_SHAPE, n))
    try:
        return rmappo_actor_params([one], [D], [1])
    except ValueError as e:
        raise ValueError("the recurrent critic must be %s: %s" % (_RCRITIC_SHAPE, e)) from None
