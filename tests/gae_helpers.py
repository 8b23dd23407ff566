"""Models of env.compute_gae (mpe_gae) for the GAE tests.

gae_mirror is the kernel's recurrence in NumPy, operation for operation: in float32 it reproduces returns and raw
advantages bit for bit (NumPy rounds every float32 operation and never fuses), and it carries a running bound on its
own float32 rounding error.  mappo_returns is a literal float64 transcription of MAPPO's
SharedReplayBuffer.compute_returns (use_gae, ValueNorm), one buffer per episode with its masks built from the episode
layout.  normalize_mirror is PPO's advantage normalisation given the (mean, std) the kernel reports."""
import numpy as np

U32 = 2.0 ** -24   # unit roundoff of float32 (round to nearest)


def _per_column(x, n):
    """(mean, std) of value_norm, [2] or [n, 2], as float32 arrays broadcasting over [n, N]"""
    x = np.asarray(x, dtype=np.float32)
    if x.ndim == 1:
        return x[0], x[1]
    return x[:, 0].reshape(n, 1), x[:, 1].reshape(n, 1)


def gae_mirror(rew, val, final, gamma, lam, episode_length=None, bootstrap=True, value_norm=None, dtype=np.float32):
    """(returns, advantages, bound) of the recurrence in mpe_b200.h over rew, val [T, n, N] and final [E, n, N] (or
    [n, N]), computed in `dtype`: np.float32 is the kernel bit for bit, np.float64 the same order in double.  gamma and
    lam are rounded to float32 first, as the kernel receives them.  bound ([T, n, N], float64) bounds |ret32 - ret| by
    the running error analysis of the float32 computation: for z = fl(x op y) with inputs carrying errors ex, ey,
    |z - exact| <= (propagated ex, ey) + u |z| / (1 - u), u = 2^-24 (the standard model of floating-point arithmetic,
    every operation rounded once).  The float32 inputs are exact; only the recurrence's roundings are bounded.

    This is a running error bound (the propagation uses the magnitudes of the mirror's own float32 intermediates) rather
    than an a-priori one written over the exact values: the a-priori form of a T-step linear recurrence, gamma_k-style,
    needs bounds on every exact intermediate before the computation and over-estimates by a factor that grows with T
    and with the cancellation in delta = (r + gamma next) - dv.  The running form follows the same standard model
    step by step and is as rigorous (|x| <= |fl(x)| / (1 - u) turns each computed magnitude into one of the exact
    value); on the tests' inputs it lies within about ten times the observed error."""
    T, n, N = rew.shape
    L = T if episode_length is None else int(episode_length)
    E = T // L
    f = dtype
    g, lm = f(np.float32(gamma)), f(np.float32(lam))
    gl = f(g * lm)
    rew, val = rew.astype(f), val.astype(f)
    final = None if final is None else np.asarray(final).reshape(E, n, N).astype(f)
    if value_norm is not None:
        mean, sd = _per_column(value_norm, n)
        mean, sd = f(mean) if np.ndim(mean) == 0 else mean.astype(f), f(sd) if np.ndim(sd) == 0 else sd.astype(f)

    q = U32 / (1.0 - U32)
    e_gl = q * abs(float(gl))                       # gl = fl(g * lm)

    def denorm(v):
        """(dv, its error bound)"""
        if value_norm is None:
            return v, np.zeros(v.shape)
        p = v * sd
        dv = p + mean
        return dv, q * np.abs(p.astype(np.float64)) + q * np.abs(dv.astype(np.float64))

    ret, adv = np.empty_like(rew), np.empty_like(rew)
    bound = np.zeros(rew.shape)
    for e in range(E - 1, -1, -1):
        if bootstrap:
            nxt, e_nxt = denorm(final[e])
        else:
            nxt, e_nxt = np.zeros((n, N), dtype=f), np.zeros((n, N))
        gae, e_gae = np.zeros((n, N), dtype=f), np.zeros((n, N))
        for t in range(e * L + L - 1, e * L - 1, -1):
            dv, e_dv = denorm(val[t])
            gn = g * nxt
            e_gn = abs(float(g)) * e_nxt + q * np.abs(gn.astype(np.float64))
            s = rew[t] + gn
            e_s = e_gn + q * np.abs(s.astype(np.float64))
            delta = s - dv
            e_delta = e_s + e_dv + q * np.abs(delta.astype(np.float64))
            c = gl * gae
            a_gae = np.abs(gae.astype(np.float64))
            e_c = abs(float(gl)) * e_gae + e_gl * (a_gae + e_gae) + q * np.abs(c.astype(np.float64))
            gae = delta + c
            e_gae = e_delta + e_c + q * np.abs(gae.astype(np.float64))
            ret[t] = gae + dv
            bound[t] = e_gae + e_dv + q * np.abs(ret[t].astype(np.float64))
            adv[t] = gae
            nxt, e_nxt = dv, e_dv
    return ret, adv, bound


def mappo_returns(rew, val, final, gamma, lam, episode_length=None, bootstrap=True, value_norm=None):
    """float64 returns of MAPPO's SharedReplayBuffer.compute_returns (use_gae; ValueNorm when value_norm is given),
    transcribed literally, run once per episode on a buffer of L steps whose value_preds[L] is the episode's final value
    (next_value) and whose masks are 1 inside the episode and masks[L] = 1 if bootstrap else 0 (the time-limit done
    zeroes it).  gamma and lam are rounded to float32 first, as the kernel receives them."""
    T, n, N = rew.shape
    L = T if episode_length is None else int(episode_length)
    E = T // L
    gamma, gae_lambda = float(np.float32(gamma)), float(np.float32(lam))
    rew, val = rew.astype(np.float64), val.astype(np.float64)
    final = np.zeros((E, n, N)) if final is None else np.asarray(final, dtype=np.float64).reshape(E, n, N)
    if value_norm is None:
        denormalize = None
    else:
        vn = np.asarray(value_norm, dtype=np.float64)
        mean, std = (vn[0], vn[1]) if vn.ndim == 1 else (vn[:, 0].reshape(n, 1), vn[:, 1].reshape(n, 1))

        def denormalize(x):
            return x * std + mean
    out = np.empty((T, n, N))
    for e in range(E):
        rewards = rew[e * L:(e + 1) * L]
        value_preds = np.concatenate([val[e * L:(e + 1) * L], final[e][None]], 0)
        masks = np.ones((L + 1, n, N))
        masks[L] = 1.0 if bootstrap else 0.0
        returns = np.zeros((L + 1, n, N))
        gae = 0
        for step in reversed(range(rewards.shape[0])):
            if denormalize is not None:
                delta = rewards[step] + gamma * denormalize(value_preds[step + 1]) * masks[step + 1] \
                    - denormalize(value_preds[step])
                gae = delta + gamma * gae_lambda * masks[step + 1] * gae
                returns[step] = gae + denormalize(value_preds[step])
            else:
                delta = rewards[step] + gamma * value_preds[step + 1] * masks[step + 1] - value_preds[step]
                gae = delta + gamma * gae_lambda * masks[step + 1] * gae
                returns[step] = gae + value_preds[step]
        out[e * L:(e + 1) * L] = returns[:L]
    return out


def normalize_mirror(adv, mean, std):
    """float32((float64(a) - mean) / (std + 1e-5)), the kernel's normalisation given its (mean, std)"""
    return ((adv.astype(np.float64) - float(mean)) / (float(std) + 1e-5)).astype(np.float32)


def seeded_inputs(T, n, N, E=1, seed=0, per_agent_norm=False):
    """float32 rewards, values [T, n, N], final values [E, n, N] and a ValueNorm (mean, std) ([2] or [n, 2]) in
    MPE-like ranges"""
    rng = np.random.RandomState(seed)
    rew = (rng.standard_normal((T, n, N)) * 0.5 - 1.0).astype(np.float32)
    val = rng.standard_normal((T, n, N)).astype(np.float32)
    final = rng.standard_normal((E, n, N)).astype(np.float32)
    shape = (n, 2) if per_agent_norm else (2,)
    vn = np.empty(shape, dtype=np.float32)
    vn[..., 0] = rng.uniform(-20.0, -5.0, shape[:-1])
    vn[..., 1] = rng.uniform(2.0, 8.0, shape[:-1])
    return rew, val, final, vn
