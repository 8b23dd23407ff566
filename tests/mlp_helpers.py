"""NumPy models of the two-hidden-layer in-kernel actor (env.rollout_policy with a Linear-ReLU-Linear-ReLU-Linear
policy): TF32 rounding as cvt.rna.tf32.f32 does it, Philox4x32-10, the Gumbel noise stream, and a float64 evaluation
of the actor with or without the kernel's operand rounding."""
import numpy as np

EXPLORE_TAG = 0x40000000


def tf32_rna(x):
    """fp32 -> TF32 (10 explicit mantissa bits) rounded to nearest, ties away from zero, returned as float32.  Adding
    half a TF32 unit to the magnitude bits and truncating rounds ties away from zero; a mantissa carry moves into the
    exponent as it should.  Inf and NaN pass unchanged."""
    b = np.asarray(x, dtype=np.float32).view(np.uint32)
    r = ((b.astype(np.uint64) + 0x1000) & 0xFFFFE000).astype(np.uint32)
    special = (b & 0x7F800000) == 0x7F800000
    return np.where(special, b, r).view(np.float32)


def philox4x32_10(ctr, key):
    """Philox4x32-10 (Salmon et al., SC'11): ctr uint32 [..., 4], key (k0, k1) -> uint32 [..., 4]"""
    M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
    mask = np.uint64(0xFFFFFFFF)
    ctr = np.asarray(ctr, dtype=np.uint64)
    c = [ctr[..., j] for j in range(4)]
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    for _ in range(10):
        p0 = np.uint64(M0) * c[0]
        p1 = np.uint64(M1) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & mask, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & mask]
        k0 = (k0 + np.uint64(W0)) & mask
        k1 = (k1 + np.uint64(W1)) & mask
    return np.stack(c, -1).astype(np.uint32)


def uniform_from_bits(bits):
    """u = ((bits >> 8) + 0.5) * 2^-24 with the sum rounded toward zero in fp32: exact below 2^23, above it the half
    does not fit in 24 bits and is dropped.  float32 in [2^-25, 1 - 2^-24]."""
    m = (np.asarray(bits, dtype=np.uint32) >> 8).astype(np.float64)
    s = np.where(m < 2 ** 23, m + 0.5, m)
    return (s * 2.0 ** -24).astype(np.float32)


def gumbel_noise(seed, epoch, world_index, t, agent, n_agents):
    """-log(-log u) of the five movement logits of `agent` at step `t` for the given global world indices, float64"""
    gw = np.asarray(world_index, dtype=np.uint64)
    key = (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    base = EXPLORE_TAG | ((t * n_agents + agent) * 2)
    words = []
    for b in (0, 1):
        ctr = np.stack([gw & np.uint64(0xFFFFFFFF), gw >> np.uint64(32), np.full_like(gw, epoch & 0xFFFFFFFF),
                        np.full_like(gw, base | b)], -1)
        words.append(philox4x32_10(ctr, key))
    bits = np.concatenate([words[0], words[1][:, :1]], 1)
    u = uniform_from_bits(bits).astype(np.float64)
    return -np.log(-np.log(u))


def actor_logits(obs, W1, b1, W2, b2, W3, b3, tf32=True):
    """float64 logits of the actor.  tf32=True rounds every tensor-core operand (observations, h1, h2, weights) to TF32
    as the kernel does; tf32=False evaluates the fp32 weights exactly."""
    f64 = np.float64
    rnd = tf32_rna if tf32 else (lambda a: np.asarray(a, dtype=np.float32))
    h1 = np.maximum(rnd(obs).astype(f64) @ rnd(W1).astype(f64).T + np.asarray(b1, f64), 0.0)
    h2 = np.maximum(rnd(h1).astype(f64) @ rnd(W2).astype(f64).T + np.asarray(b2, f64), 0.0)
    return rnd(h2).astype(f64) @ rnd(W3).astype(f64).T + np.asarray(b3, f64)


def softmax(z):
    e = np.exp(z - z.max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)
