"""NumPy models of rMAPPO's recurrent centralized critic (env.rollout_policy(rmappo_actors, T, critic=(base, gru, norm,
v_out)), mpe_critic_gru): the kernel's recipe is the recurrent actor's (RecurrentModel) on share_obs with a [1, 64]
head, so this module adds only the critic's pieces -- seeded critics, the written bound on a value given the kernel's
own h', the free-running float64 evaluation of the user's modules over a whole rollout, and the mirror of the kernels'
block table (kRCriticWarps in csrc/mpe_kernels.cu)."""
import numpy as np

from mappo_helpers import layer_norm, norm_error_bound
from mlp_helpers import tf32_accumulation_bound
from rmappo_helpers import H, TF32_ULP, RecurrentModel, make_rmappo_actor, module_step

# the programs the recurrent critic is built for (GruBuilt) and its block size (kRCriticWarps)
RCRITIC_PROGRAMS = ("simple", "simple_spread_n2", "simple_spread_n3", "simple_spread_n4", "simple_spread_n5",
                    "simple_spread_n6", "simple_reference")
RCRITIC_WARPS = 8
# against the unfolded float64 critic run free from h0 over T = 25 steps every value stays within LOOSE
LOOSE = 2e-2


def make_rcritic(obs_dims, tanh, feature_norm, seed=7, eps=1e-5, device="cuda"):
    """one seeded (base, gru, norm, v_out) over share_obs (D = sum(obs_dims)), shaped as the recurrent actor"""
    return make_rmappo_actor(int(sum(obs_dims)), 1, tanh, feature_norm, seed=seed, eps=eps, device=device)


def value_bound(model, hn):
    """Per-row bound on |kernel V - model.logits(hn)| for the kernel's own h' [m, 64]: the fp32 tensor-core sum of the
    64 TF32 terms of v_out, a few ulps of V, and the TF32 flips LN(h') may take (the kernel's fp32 LayerNorm within
    norm_error_bound of the float64 one, then one TF32 ulp): sum_j |w3_j| 2^-10 (|LN(h')_j| + norm error)."""
    hn = np.asarray(hn, np.float64)
    x = model.rnd(layer_norm(hn, model.eps))
    v = x @ model.W[4].T + model.b[4]
    flips = (TF32_ULP * (np.abs(layer_norm(hn, model.eps)) + norm_error_bound(hn, np.zeros_like(hn), model.eps))) @ \
        np.abs(model.W[4]).T
    return (tf32_accumulation_bound(x, model.W[4], model.b[4]) + flips + 4 * 2.0 ** -24 * np.abs(v))[:, 0]


def module_rollout(critic, share_obs, final_obs, h0, episode_length=None):
    """the user's unfolded critic in float64, run free over share_obs [T, N, D] from h0 [N, 64] (zeros at every
    episode's start when episode_length is given): (values [T, N], final values [E, N], h after the last step)"""
    T = share_obs.shape[0]
    L = episode_length or T
    h = np.asarray(h0, np.float64)
    values, finals = [], []
    for t in range(T):
        if episode_length and t % L == 0:
            h = np.zeros_like(h)
        v, h = module_step(critic, share_obs[t], h)
        values.append(v[:, 0])
        if (t + 1) % L == 0 and (episode_length or t == T - 1):
            finals.append(module_step(critic, final_obs[t // L], h)[0][:, 0])
    return np.stack(values), np.stack(finals), h


__all__ = ["H", "LOOSE", "RCRITIC_PROGRAMS", "RCRITIC_WARPS", "RecurrentModel", "make_rcritic", "module_rollout",
           "value_bound"]
