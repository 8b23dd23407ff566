"""NativeWorld: the batch state tensors of one World plus the libmpe_b200 handle that steps them.

PyTorch owns every buffer (device memory, pinned host memory, streams); the library borrows raw
pointers per call (include/mpe_b200.h).  Nothing in this module computes: it allocates, packs
pointers and launches.  A missing extension or a machine without a CUDA device raises.
"""
import ctypes

import numpy as np

from . import _lib
from ._lib import check


def _align(x, a=256):
    return (x + a - 1) // a * a


class ShapeHandle(object):
    """Device-less handle (mpe_create(..., device=-1)): validates the descriptor against its
    compiled program and answers the shape queries MultiAgentEnv.__init__ needs
    (environment.py:39-70).  Works on machines without a GPU."""

    def __init__(self, desc, n_env, device_index=-1):
        self.lib = _lib.load()
        self.desc = desc
        self.n_env = int(n_env)
        h = ctypes.c_void_p()
        check(self.lib.mpe_create(ctypes.byref(desc), self.n_env, device_index, ctypes.byref(h)), "mpe_create")
        self.handle = h
        lib = self.lib
        self.n_agents = lib.mpe_num_agents(h)
        self.n_landmarks = int(desc.n_landmarks)
        self.dim_c = int(desc.dim_c)
        self.custom = int(desc.scenario) == _lib.SCN_CUSTOM     # observation / reward live in the user's torch code
        self.obs_dims = [] if self.custom else [lib.mpe_obs_dim(h, i) for i in range(self.n_agents)]
        self.act_dims = [lib.mpe_act_dim(h, i) for i in range(self.n_agents)]
        self.n_speakers = lib.mpe_num_speakers(h)
        self.n_goals = lib.mpe_num_goals(h)
        self.info_dim = lib.mpe_info_dim(h)
        self.bytes_per_env_step = lib.mpe_bytes_per_env_step(h)
        self._speakers = [i for i in range(self.n_agents) if not desc.agent_silent[i]]

    def gru_separated_workspace_bytes(self):
        """bytes of the per-agent recurrent actors' workspace, every agent's fragment image
        (mpe_rollout_policy_gru_separated_workspace_bytes); MpeError for a program without them.  Needs no device."""
        return check(self.lib.mpe_rollout_policy_gru_separated_workspace_bytes(self.handle),
                     "mpe_rollout_policy_gru_separated_workspace_bytes")

    def require_gru_separated(self):
        """MpeError unless the library has per-agent recurrent actors and critics (rMAPPO's separated runner) for this
        program.  The device-less workspace query answers it."""
        self.gru_separated_workspace_bytes()

    def speaker_slot(self, agent_index):
        """row block of agent `agent_index` in the comm tensors, or -1 if the agent is silent"""
        try:
            return self._speakers.index(agent_index)
        except ValueError:
            return -1

    def close(self):
        if getattr(self, "handle", None) is not None and self.handle.value:
            self.lib.mpe_destroy(self.handle)
            self.handle = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001  (interpreter shutdown)
            pass


class Outputs(object):
    """One slab holding everything a step produces, so that a host caller gets it with a single
    DMA: obs_0 | obs_1 | ... | rew [A][N] | done [A][N] | info [A][INFO][N] (256-byte aligned parts;
    mpe_step_host coalesces the adjacent parts into one cudaMemcpyAsync)."""

    def __init__(self, nw, pinned_host=False):
        import torch
        N, A = nw.n_env, nw.n_agents
        offs, off = [], 0
        for od in nw.obs_dims:
            offs.append(off)
            off = _align(off + N * od * 4)
        rew_off = off
        off = _align(off + A * N * 4)
        done_off = off
        off = _align(off + A * N)
        info_off = off
        off = _align(off + A * nw.info_dim * N * 4)
        if pinned_host:
            self.slab = torch.empty(off, dtype=torch.uint8, pin_memory=True)
        else:
            self.slab = torch.empty(off, dtype=torch.uint8, device=nw.device)
        s = self.slab
        self.obs = [s[o:o + N * od * 4].view(torch.float32).view(N, od) for o, od in zip(offs, nw.obs_dims)]
        self.rew = s[rew_off:rew_off + A * N * 4].view(torch.float32).view(A, N)
        self.info = None
        if nw.info_dim > 0:
            self.info = s[info_off:info_off + A * nw.info_dim * N * 4].view(torch.float32).view(A, nw.info_dim, N)
        self.done = s[done_off:done_off + A * N].view(A, N)
        # per-agent views handed to the caller (built once: persistent outputs are reused every step)
        self.rew_list = [self.rew[i] for i in range(A)]
        done_b = self.done.view(torch.bool)
        self.done_list = [done_b[i] for i in range(A)]
        if pinned_host:   # NumPy views of the same pinned memory (scalar convention: no per-step tensor ops)
            self.obs_np = [o.numpy() for o in self.obs]
            self.rew_np, self.done_np = self.rew.numpy(), self.done.numpy()
            self.info_np = self.info.numpy() if self.info is not None else None
        self.obs_ptrs = _lib.ptr_array([t.data_ptr() for t in self.obs])
        self.rew_ptr = self.rew.data_ptr()
        self.done_ptr = self.done.data_ptr()
        self.info_ptr = self.info.data_ptr() if self.info is not None else None


class FreshOutputs(object):
    """Per-step device outputs for callers that keep what `step` returns (the reference hands out freshly
    allocated arrays).  Same attributes as `Outputs`, built with as few tensor operations as possible -- one
    float slab carved with as_strided, `unbind` for the per-agent views -- because at ~6 us per kernel the
    host-side cost of a step is what a GPU-resident trainer actually waits for."""

    def __init__(self, nw):
        import torch
        N, A = nw.n_env, nw.n_agents
        lay = nw._fresh_layout
        fs = torch.empty(lay["words"], dtype=torch.float32, device=nw.device)
        self.slab = fs
        self.obs = [fs.as_strided((N, od), (od, 1), off) for off, od in lay["obs"]]
        self.rew = fs.as_strided((A, N), (N, 1), lay["rew"])
        self.rew_list = self.rew.unbind(0)
        self.info = fs.as_strided((A, nw.info_dim, N), (nw.info_dim * N, N, 1), lay["info"]) if nw.info_dim > 0 else None
        done_b = torch.empty((A, N), dtype=torch.bool, device=nw.device)   # written as 0/1 bytes by the kernel
        self.done = done_b.view(torch.uint8)
        self.done_list = done_b.unbind(0)
        base = fs.data_ptr()
        self.obs_ptrs = _lib.ptr_array([base + 4 * off for off, _ in lay["obs"]])
        self.rew_ptr = base + 4 * lay["rew"]
        self.done_ptr = done_b.data_ptr()
        self.info_ptr = base + 4 * lay["info"] if nw.info_dim > 0 else None


class NativeWorld(ShapeHandle):
    def __init__(self, desc, n_env, device=None, seed=0, world_offset=0):
        import torch
        if not torch.cuda.is_available():
            raise RuntimeError("multiagent_particle_envs_b200 needs a CUDA device (H100, sm_90a); "
                               "there is no CPU fallback")
        self.torch = torch
        dev = torch.device(device if device is not None else "cuda")
        if dev.type != "cuda":
            raise RuntimeError("device must be a CUDA device, got %s" % (dev,))
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        self.device = dev
        super(NativeWorld, self).__init__(desc, n_env, dev.index)
        N, A, L = self.n_env, self.n_agents, self.n_landmarks
        NC = self.n_speakers * self.dim_c
        f32 = dict(dtype=torch.float32, device=dev)
        # ---- state, struct-of-arrays over worlds (include/mpe_b200.h) ----
        self.agent_pv = torch.zeros(A, N, 4, **f32)
        self.lm_p = torch.zeros(max(L, 1), N, 2, **f32)
        self.comm = torch.zeros(max(NC, 1), N, **f32)
        self.goal = torch.zeros(max(self.n_goals, 1), N, dtype=torch.int32, device=dev)
        # ---- decoded actions for World.step() ----
        self.act_u = torch.zeros(A, N, 2, **f32)
        self.act_c = torch.zeros(max(NC, 1), N, **f32)
        self.seed = int(seed)
        self.world_offset = int(world_offset)
        self.epoch = 0
        self._epoch_dev = None
        # layout of FreshOutputs' float slab, in 4-byte words (every part 64-word = 256-byte aligned)
        off, obs_l = 0, []
        for od in self.obs_dims:
            obs_l.append((off, od))
            off = _align(off + N * od, 64)
        rew_off = off
        off = _align(off + A * N, 64)
        info_off = off
        off = _align(off + A * self.info_dim * N, 64)
        self._fresh_layout = dict(obs=obs_l, rew=rew_off, info=info_off, words=max(off, 64))
        self.out = None if self.custom else Outputs(self)   # persistent outputs (reset / step in reuse mode)
        self.cb_out = None                 # lazily created: outputs of direct scenario-callback calls (core.py)
        self._host = None                  # lazily created staging for host callers
        self._has_comm = NC > 0
        self._has_goal = self.n_goals > 0

    # ---- helpers ---------------------------------------------------------------------------
    def _stream(self):
        return ctypes.c_void_p(self.torch.cuda.current_stream(self.device).cuda_stream)

    def _state_ptrs(self):
        return (self.agent_pv.data_ptr(), self.lm_p.data_ptr(),
                self.comm.data_ptr() if self._has_comm else None,
                self.goal.data_ptr() if self._has_goal else None)

    def new_outputs(self):
        return FreshOutputs(self)

    def persistent_outputs(self):
        return Outputs(self)

    # ---- reset -------------------------------------------------------------------------------
    def reset(self, mask=None):
        torch = self.torch
        mptr = None
        if mask is not None:
            mask = torch.as_tensor(mask, device=self.device).to(torch.uint8).contiguous()
            if mask.numel() != self.n_env:
                raise ValueError("reset mask must have one entry per world")
            mptr = mask.data_ptr()
        pv, lm, comm, goal = self._state_ptrs()
        if self.torch.cuda.is_current_stream_capturing():
            # inside a CUDA-graph capture the epoch must live on the device, or every replay would redraw the
            # same initial conditions
            if self._epoch_dev is None:
                raise RuntimeError("call NativeWorld.enable_device_epoch() before capturing a reset in a CUDA graph")
            check(self.lib.mpe_reset_dev_epoch(self.handle, pv, lm, comm, goal, mptr, self.seed, self.world_offset,
                                               self._epoch_dev.data_ptr(), self._stream()), "mpe_reset_dev_epoch")
            return
        if self._epoch_dev is not None:
            self.epoch = int(self._epoch_dev.item())
        check(self.lib.mpe_reset(self.handle, pv, lm, comm, goal, mptr, self.seed, self.world_offset,
                                 self.epoch, self._stream()), "mpe_reset")
        self.epoch += 1
        if self._epoch_dev is not None:
            self._epoch_dev.fill_(self.epoch)

    def enable_device_epoch(self):
        """keep the reset epoch in device memory so that resets captured in CUDA graphs advance it on replay"""
        if self._epoch_dev is None:
            self._epoch_dev = self.torch.full((1,), self.epoch, dtype=self.torch.int64, device=self.device)
        return self._epoch_dev

    # ---- the hot path ------------------------------------------------------------------------
    def set_action(self, act_ptrs, flags=0):
        check(self.lib.mpe_set_action(self.handle, act_ptrs, self.act_u.data_ptr(),
                                      self.act_c.data_ptr() if self._has_comm else None,
                                      flags & ~_lib.FLAG_SHARED_REWARD, self._stream()), "mpe_set_action")

    def world_step(self):
        pv, lm, comm, _ = self._state_ptrs()
        check(self.lib.mpe_world_step(self.handle, pv, lm, comm, self.act_u.data_ptr(),
                                      self.act_c.data_ptr() if self._has_comm else None, self._stream()),
              "mpe_world_step")

    def observe(self, out=None, flags=0, with_info=True):
        out = out or self.out
        pv, lm, comm, goal = self._state_ptrs()
        check(self.lib.mpe_observe(self.handle, pv, lm, comm, goal, out.obs_ptrs, out.rew_ptr, out.done_ptr,
                                   out.info_ptr if with_info else None, flags, self._stream()), "mpe_observe")
        return out

    def step(self, act_ptrs, out=None, flags=0, with_info=False):
        """MultiAgentEnv.step fused into one launch; act_ptrs: ctypes array of device pointers.
        benchmark_data (info) is computed and written only when asked for (make_env(benchmark=True))."""
        out = out or self.out
        pv, lm, comm, goal = self._state_ptrs()
        check(self.lib.mpe_step(self.handle, pv, lm, comm, goal, act_ptrs, out.obs_ptrs, out.rew_ptr,
                                out.done_ptr, out.info_ptr if with_info else None, flags, self._stream()),
              "mpe_step")
        return out

    def rollout(self, act_seq_ptrs, n_steps, out=None, flags=0, rew_steps=None):
        """n_steps fused steps on pre-generated actions in ONE launch (mpe_rollout): the state stays in registers
        between the steps.  out.obs / out.done describe the final state, out.rew holds the summed rewards;
        rew_steps: optional float32 [n_steps, A, N] CUDA tensor receiving every step's rewards."""
        out = out or self.out
        pv, lm, comm, goal = self._state_ptrs()
        check(self.lib.mpe_rollout(self.handle, pv, lm, comm, goal, act_seq_ptrs, int(n_steps), out.obs_ptrs, out.rew_ptr,
                                   rew_steps.data_ptr() if rew_steps is not None else None, out.done_ptr, flags,
                                   self._stream()), "mpe_rollout")
        return out

    def rollout_policy(self, w1_ptrs, b1_ptrs, w2_ptrs, b2_ptrs, hidden, n_steps, out=None, flags=0, rew_steps=None,
                       act_rec_ptrs=None):
        """n_steps fused steps in ONE launch with every agent's two-layer perceptron evaluated inside the kernel
        (mpe_rollout_policy); pointer arrays hold one device pointer per agent."""
        out = out or self.out
        pv, lm, comm, goal = self._state_ptrs()
        check(self.lib.mpe_rollout_policy(self.handle, pv, lm, comm, goal, w1_ptrs, b1_ptrs, w2_ptrs, b2_ptrs, int(hidden),
                                          int(n_steps), out.obs_ptrs, out.rew_ptr,
                                          rew_steps.data_ptr() if rew_steps is not None else None, act_rec_ptrs,
                                          out.done_ptr, flags, self._stream()), "mpe_rollout_policy")
        return out

    def require_mlp_actor(self):
        """MpeError unless the library has the two-hidden-layer actor for this program.  mpe_rollout_policy_mlp checks
        the program before any pointer, so a call without state or weights answers that and runs nothing."""
        none = _lib.ptr_array([None] * self.n_agents)
        rc = self.lib.mpe_rollout_policy_mlp(self.handle, None, None, None, None, none, none, none, none, none, none, 32,
                                             0, 0, 0, 0, 0, None, None, None, None, None, None, 0, self._stream())
        if rc == _lib.ERR_UNSUPPORTED:
            check(rc, "mpe_rollout_policy_mlp")

    def require_gru_actor(self):
        """MpeError unless the library has MAPPO's recurrent actor for this program.  As in require_mlp_actor, the probe
        reaches the program check and stops at the null state: the aligned dummy weight addresses are never read."""
        rc = self.lib.mpe_rollout_policy_gru(self.handle, None, None, None, None, *([256] * 10), 64, 0, 0, 0, 0, 0,
                                             None, None, None, None, None, None, None, None, 0, 0.0, None, 0,
                                             self._stream())
        if rc == _lib.ERR_UNSUPPORTED:
            check(rc, "mpe_rollout_policy_gru")

    def require_critic(self, count):
        """MpeError unless the library has MAPPO's critic kernel for this program and `count` critics (1 or A) fit in
        shared memory next to the actor.  As in require_gru_actor, the probe stops at the null state."""
        none = _lib.ptr_array([256] * self.n_agents)
        rc = self.lib.mpe_rollout_policy_mappo_critic(self.handle, None, None, None, None, *([none] * 6), 64, 0, 0, 0, 0,
                                                      0, None, None, None, None, None, None, 0, 0.0, int(count),
                                                      *([none] * 6), None, None, None, 0, self._stream())
        if rc == _lib.ERR_UNSUPPORTED:
            check(rc, "mpe_rollout_policy_mappo_critic")

    def require_local_critic(self, count):
        """MpeError unless the library has IPPO's local critics next to MAPPO's actor for this program and `count`
        critics (1 or A) fit in shared memory.  As in require_critic, the probe stops at the null state."""
        none = _lib.ptr_array([256] * self.n_agents)
        rc = self.lib.mpe_rollout_policy_mappo_local_critic(self.handle, None, None, None, None, *([none] * 6), 64, 0, 0,
                                                            0, 0, 0, None, None, None, None, None, None, 0, 0.0,
                                                            int(count), *([none] * 6), None, None, None, 0,
                                                            self._stream())
        if rc == _lib.ERR_UNSUPPORTED:
            check(rc, "mpe_rollout_policy_mappo_local_critic")

    def require_critic_gru_local(self):
        """MpeError unless the library has rIPPO's recurrent local critic for this program (probed as
        require_critic_gru)."""
        rc = self.lib.mpe_critic_gru_local(self.handle, None, None, 0, 0, *([256] * 10), None, None, None, None, 0, 0.0,
                                           self._stream())
        if rc == _lib.ERR_UNSUPPORTED:
            check(rc, "mpe_critic_gru_local")

    def require_critic_gru(self):
        """MpeError unless the library has rMAPPO's recurrent critic for this program.  mpe_critic_gru checks the program
        before any pointer, so the probe stops at the null state and runs nothing."""
        rc = self.lib.mpe_critic_gru(self.handle, None, None, 0, 0, *([256] * 10), None, None, None, None, 0, 0.0,
                                     self._stream())
        if rc == _lib.ERR_UNSUPPORTED:
            check(rc, "mpe_critic_gru")

    def critic_gru(self, w_ptrs, obs_rec_ptrs, final_obs_ptrs, n_steps, episode_length, rnn_state, rnn_record, values,
                   final_values, net, local=False):
        """rMAPPO's recurrent critic over a finished rollout's records (mpe_critic_gru), on the current stream: w_ptrs
        the ten device pointers of its folded weight set (environment.rmappo_critic_params), obs_rec_ptrs and
        final_obs_ptrs one [n_steps, N, obs_dim_i] and one [E, N, obs_dim_i] record per agent, episode_length None
        (one episode) or L.  rnn_state (float32 [N, 64]) holds the initial h (unless episode_length) and receives the
        final one, rnn_record (float32 [n_steps, N, 64] or None) the h each step consumed; values [n_steps, A, N] and
        final_values [E, A, N] receive the values.  net = (net_flags, eps) as in rollout_policy_mlp.  local=True
        (mpe_critic_gru_local): rIPPO's local critic, its W1 [64, obs_dim], run on every agent's own records with
        rnn_state [A, N, 64] and rnn_record [n_steps, A, N, 64], agent k's values in row k."""
        name = "mpe_critic_gru_local" if local else "mpe_critic_gru"
        rc = getattr(self.lib, name)(self.handle, obs_rec_ptrs, final_obs_ptrs, int(n_steps), int(episode_length or 0),
                                     *w_ptrs, rnn_state.data_ptr(), rnn_record.data_ptr() if rnn_record is not None
                                     else None, values.data_ptr(), final_values.data_ptr(), int(net[0]), float(net[1]),
                                     self._stream())
        check(rc, name)

    def critic_gru_separated(self, w_ptrs, obs_rec_ptrs, final_obs_ptrs, n_steps, episode_length, rnn_state, rnn_record,
                             values, final_values, net):
        """rMAPPO's per-agent recurrent critics (mpe_critic_gru_separated) as critic_gru, but w_ptrs are ten pointer
        arrays (critic k's weight at entry k), rnn_state is float32 [A, N, 64] and rnn_record [n_steps, A, N, 64] or
        None, and critic k writes only agent k's values."""
        rc = self.lib.mpe_critic_gru_separated(self.handle, obs_rec_ptrs, final_obs_ptrs, int(n_steps),
                                               int(episode_length or 0), *w_ptrs, rnn_state.data_ptr(),
                                               rnn_record.data_ptr() if rnn_record is not None else None,
                                               values.data_ptr(), final_values.data_ptr(), int(net[0]), float(net[1]),
                                               self._stream())
        check(rc, "mpe_critic_gru_separated")

    def gae_workspace_bytes(self):
        """bytes of the workspace gae needs to normalise the advantages (mpe_gae_workspace_bytes)"""
        return check(self.lib.mpe_gae_workspace_bytes(self.handle), "mpe_gae_workspace_bytes")

    def gae(self, rewards, values, final_values, n_steps, episode_length, gamma, gae_lambda, flags, value_norm, returns,
            advantages, workspace):
        """MAPPO's GAE and returns (mpe_gae) on the current stream: rewards, values, returns, advantages float32
        [n_steps, A, N], final_values [E, A, N] (or None without _lib.GAE_BOOTSTRAP), episode_length None (one
        episode) or L, value_norm None or float32 (mean, std) [2] / [A, 2], workspace None or a tensor of at least
        gae_workspace_bytes() bytes (with _lib.GAE_NORMALIZE; it then starts with the float64 (mean, std))."""
        ptr = lambda t: t.data_ptr() if t is not None else None   # noqa: E731
        rc = self.lib.mpe_gae(self.handle, rewards.data_ptr(), values.data_ptr(), ptr(final_values), int(n_steps),
                              int(episode_length or 0), float(gamma), float(gae_lambda), int(flags), ptr(value_norm),
                              returns.data_ptr(), advantages.data_ptr(), ptr(workspace),
                              workspace.numel() * workspace.element_size() if workspace is not None else 0,
                              self._stream())
        check(rc, "mpe_gae")

    def rollout_policy_mlp(self, w_ptrs, hidden, n_steps, out=None, flags=0, *, episode_length=None, categorical=False,
                           rew_steps=None, act_rec_ptrs=None, obs_rec_ptrs=None, final_obs_ptrs=None, logp_steps=None,
                           ep_rew=None, explore_seed=None, explore_epoch=0, mappo=None, gru=None, critic=None,
                           local_critic=False):
        """n_steps fused steps in ONE launch with every agent's two-hidden-layer actor evaluated on the tensor cores
        (mpe_rollout_policy_mlp); w_ptrs: the six pointer arrays (W1, b1, W2, b2, W3, b3), one device pointer per
        agent each.  explore_seed (not None) switches the Gumbel-softmax sampling on.

        categorical=True (mpe_rollout_policy_mlp_categorical): every agent applies the one-hot vector of the arg-max per
        sub-space, of the Gumbel-perturbed logits when exploring; act_rec_ptrs then holds one int32 [n_steps, N, n_sub_i]
        index record per agent, and logp_steps (float32 [n_steps, A, N]) receives the log-probabilities.

        episode_length=L (mpe_rollout_policy_mlp[_categorical]_episodes): n_steps / L episodes, and after each episode
        the reset that `reset()` would draw, inside the kernel.  The resets use the epochs `reset()` would use next, and
        self.epoch (and the device epoch, if enabled) advances by the number of episodes.  ep_rew: float32 [episodes, A,
        N] CUDA tensor receiving each episode's returns; out.obs receives the observations of the state after the last
        reset; final_obs_ptrs: one [episodes, N, obs_dim_i] record per agent of each episode's last observation.

        mappo=(net_flags, eps) (mpe_rollout_policy_mappo[_episodes], categorical only): MAPPO's actor, w_ptrs holding
        its folded network (environment.mappo_actor_params); net_flags is _lib.MAPPO_FEATURE_NORM | _lib.MAPPO_TANH.

        gru=(rnn_state, rnn_record) with mappo (mpe_rollout_policy_gru[_episodes]): MAPPO's recurrent actor.  w_ptrs is
        then the ten device pointers of its one shared folded weight set (W1, b1, W2, b2, W_ih, b_ih, W_hh, b_hh, W3,
        b3; environment.rmappo_actor_params); rnn_state, a float32 [A, N, 64] CUDA tensor, holds the initial hidden
        state and receives the final one, and rnn_record (float32 [n_steps, A, N, 64], or None) the h each step
        consumed.  gru=(rnn_state, rnn_record, workspace) (mpe_rollout_policy_gru_separated[_episodes]): every agent's
        own recurrent actor; w_ptrs is then ten pointer arrays, agent i's folded weight at entry i, and workspace a
        16-byte aligned CUDA tensor of at least gru_separated_workspace_bytes() bytes.

        critic=(count, cw_ptrs, values, final_values) with mappo (mpe_rollout_policy_mappo_critic[_episodes]): MAPPO's
        centralized critic next to the actor.  count is 1 (one shared critic) or A; cw_ptrs the six pointer arrays of
        the folded critics (environment.mappo_critic_params), count device pointers each; values a float32 [n_steps, A,
        N] and final_values a float32 [A, N] ([episodes, A, N]) CUDA tensor.  local_critic=True
        (mpe_rollout_policy_mappo_local_critic[_episodes]): the critics are IPPO's local ones, critic k's W1 [64,
        obs_dim_k] (one shared critic: every agent's obs_dim)."""
        out = out or self.out
        episodes = episode_length is not None
        if gru is not None and mappo is None:
            raise ValueError("rollout_policy_mlp: the recurrent actor is MAPPO's (pass mappo=(net_flags, eps))")
        if critic is not None and (mappo is None or gru is not None):
            raise ValueError("rollout_policy_mlp: the critic runs next to MAPPO's MLP actor (pass mappo, not gru)")
        if mappo is not None and not categorical:
            raise ValueError("rollout_policy_mlp: the MAPPO actor has the categorical form only")
        if episodes and self.torch.cuda.is_current_stream_capturing():
            raise RuntimeError("rollout_policy with episode_length cannot be captured in a CUDA graph: the reset epoch "
                               "is a launch argument")
        pv, lm, comm, goal = self._state_ptrs()
        explore = explore_seed is not None
        explore_args = (int(explore), int(explore_seed) if explore else 0, int(explore_epoch))
        rew_ptr = rew_steps.data_ptr() if rew_steps is not None else None
        logp = (logp_steps.data_ptr() if logp_steps is not None else None,) if categorical else ()
        rnn = ()
        if critic is not None:
            name = "mpe_rollout_policy_mappo_" + ("local_critic" if local_critic else "critic") + \
                ("_episodes" if episodes else "")
            net = (int(mappo[0]), float(mappo[1]), int(critic[0]), *critic[1], critic[2].data_ptr(),
                   critic[3].data_ptr())
        elif gru is not None:
            separated = len(gru) == 3
            name = "mpe_rollout_policy_gru" + ("_separated" if separated else "") + ("_episodes" if episodes else "")
            net = (int(mappo[0]), float(mappo[1]))
            rnn = (gru[0].data_ptr(), gru[1].data_ptr() if gru[1] is not None else None)
            if separated:
                rnn += (gru[2].data_ptr(), gru[2].numel() * gru[2].element_size())
        elif mappo is not None:
            name = "mpe_rollout_policy_mappo" + ("_episodes" if episodes else "")
            net = (int(mappo[0]), float(mappo[1]))
        else:
            name = "mpe_rollout_policy_mlp" + ("_categorical" if categorical else "") + ("_episodes" if episodes else "")
            net = ()
        if episodes:
            epoch = int(self._epoch_dev.item()) if self._epoch_dev is not None else self.epoch
            n_episodes = int(n_steps) // int(episode_length)
            rc = getattr(self.lib, name)(self.handle, pv, lm, comm, goal, *w_ptrs, int(hidden), int(episode_length),
                                         n_episodes, *explore_args, self.seed, epoch, self.world_offset, out.obs_ptrs,
                                         ep_rew.data_ptr(), rew_ptr, *logp, act_rec_ptrs, obs_rec_ptrs, final_obs_ptrs,
                                         *rnn, *net, out.done_ptr, flags, self._stream())
        else:
            rc = getattr(self.lib, name)(self.handle, pv, lm, comm, goal, *w_ptrs, int(hidden), int(n_steps), *explore_args,
                                         self.world_offset, out.obs_ptrs, out.rew_ptr, rew_ptr, *logp, act_rec_ptrs,
                                         obs_rec_ptrs, *rnn, *net, out.done_ptr, flags, self._stream())
        check(rc, name)
        if episodes:
            self.epoch = epoch + n_episodes
            if self._epoch_dev is not None:
                self._epoch_dev.fill_(self.epoch)
        return out

    # ---- host callers (what the reference's callers hold: NumPy arrays) -----------------------
    def host_staging(self):
        if self._host is None:
            torch = self.torch
            N = self.n_env
            host_act = [torch.zeros(N, ad, dtype=torch.float32).pin_memory() for ad in self.act_dims]
            dev_act = [torch.zeros(N, ad, dtype=torch.float32, device=self.device) for ad in self.act_dims]
            self._host = dict(
                host_act=host_act, dev_act=dev_act, host_act_np=[t.numpy() for t in host_act],
                host_act_ptrs=_lib.ptr_array([t.data_ptr() for t in host_act]),
                dev_act_ptrs=_lib.ptr_array([t.data_ptr() for t in dev_act]),
                host_out=[Outputs(self, pinned_host=True), Outputs(self, pinned_host=True)], flip=0)
        return self._host

    def step_host(self, host_act_ptrs, flags=0, dev_out=None, host_out=None, with_info=False):
        """H2D actions -> fused step -> D2H outputs, all enqueued on the current stream by
        mpe_step_host; returns the pinned host Outputs (valid after a stream synchronize)."""
        hs = self.host_staging()
        dev_out = dev_out or self.out
        if host_out is None:
            host_out = hs["host_out"][hs["flip"]]
            hs["flip"] ^= 1
        pv, lm, comm, goal = self._state_ptrs()
        check(self.lib.mpe_step_host(self.handle, pv, lm, comm, goal, host_act_ptrs, hs["dev_act_ptrs"],
                                     dev_out.obs_ptrs, dev_out.rew_ptr, dev_out.done_ptr,
                                     dev_out.info_ptr if with_info else None,
                                     host_out.obs_ptrs, host_out.rew_ptr, host_out.done_ptr,
                                     host_out.info_ptr if with_info else None,
                                     flags | _lib.FLAG_HOST_SLAB, self._stream()), "mpe_step_host")
        return host_out

    # ---- benchmark_data (e.g. simple_spread.py:47-63) -----------------------------------------
    def benchmark_data(self, i, batched, out=None):
        """scenario.benchmark_data(agent i) from the info channel, in the reference's return shape"""
        out = out or self.out
        sc = self.desc.scenario
        if out.info is None:
            return {}
        info = out.info[i]                     # [info_dim, N]
        adv = bool(self.desc.agent_adversary[i])
        L, C = self.n_landmarks, self.dim_c
        if batched:
            if sc == _lib.SCN_SPREAD:           # (rew, collisions, min_dists, occupied_landmarks)
                return (info[0], info[1], info[2], info[3])
            if sc == _lib.SCN_ADVERSARY:        # adversary: |p - goal|^2; good: (|p - lm_l|^2 ..., |p - goal|^2)
                return info[0] if adv else tuple(info[q] for q in range(L + 1))
            if sc == _lib.SCN_CRYPTO:           # (agent.state.c, goal colour)
                return (info[0:C].t(), info[C:2 * C].t())
            return info[0]
        v = (out.info_np[i, :, 0] if getattr(out, "info_np", None) is not None
             else info[:, 0].detach().to("cpu").numpy()).astype(np.float64)
        if sc == _lib.SCN_SPREAD:
            return (float(v[0]), int(v[1]), float(v[2]), int(v[3]))
        if sc == _lib.SCN_ADVERSARY:
            return float(v[0]) if adv else tuple(float(x) for x in v[:L + 1])
        if sc == _lib.SCN_CRYPTO:
            return (v[0:C].copy(), v[C:2 * C].copy())
        return int(v[0])
