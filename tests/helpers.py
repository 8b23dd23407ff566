"""shared test helpers (the oracle is imported HERE, in tests/, only as the checker)"""
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# golden tag -> (scenario name, scenario kwargs)
CONFIGS = {
    "simple": ("simple", {}),
    "simple_spread_n3": ("simple_spread", {}),
    "simple_spread_n6": ("simple_spread", {"num_agents": 6}),
    "simple_tag": ("simple_tag", {}),
    "simple_world_comm": ("simple_world_comm", {}),
    "simple_adversary": ("simple_adversary", {}),
    "simple_push": ("simple_push", {}),
    "simple_speaker_listener": ("simple_speaker_listener", {}),
    "simple_reference": ("simple_reference", {}),
    "simple_crypto": ("simple_crypto", {}),
}
# entity-count variants the reference hard-codes away (their goldens build the world test-side, oracle/refshim.py)
VARIANTS = {
    "simple_spread_n2": ("simple_spread", {"num_agents": 2}),
    "simple_spread_n4": ("simple_spread", {"num_agents": 4}),
    "simple_spread_n5": ("simple_spread", {"num_agents": 5}),
    "simple_tag_1v1": ("simple_tag", {"num_adversaries": 1, "num_good_agents": 1, "num_landmarks": 2}),
    "simple_tag_2v1": ("simple_tag", {"num_adversaries": 2, "num_good_agents": 1, "num_landmarks": 2}),
    "simple_tag_4v2": ("simple_tag", {"num_adversaries": 4, "num_good_agents": 2, "num_landmarks": 2}),
    "simple_tag_6v2": ("simple_tag", {"num_adversaries": 6, "num_good_agents": 2, "num_landmarks": 3}),
    "simple_adversary_n4": ("simple_adversary", {"num_agents": 4}),
}
NO_BENCHMARK = ("simple", "simple_push", "simple_speaker_listener", "simple_reference")
# every program the library compiles (csrc/mpe_kernels.cu programs()), one tag each
PROGRAM_TAGS = list(CONFIGS) + list(VARIANTS)
assert len(PROGRAM_TAGS) == 18
# the program types of csrc/mpe_kernels.cu (make_program), as c++filt prints them
TYPE_TAGS = {
    "Simple<1, 1>": "simple", "Spread<2>": "simple_spread_n2", "Spread<3>": "simple_spread_n3",
    "Spread<4>": "simple_spread_n4", "Spread<5>": "simple_spread_n5", "Spread<6>": "simple_spread_n6",
    "Tag<3, 1, 2>": "simple_tag", "Tag<1, 1, 2>": "simple_tag_1v1", "Tag<2, 1, 2>": "simple_tag_2v1",
    "Tag<4, 2, 2>": "simple_tag_4v2", "Tag<6, 2, 3>": "simple_tag_6v2", "WorldComm<4, 2, 1, 2>": "simple_world_comm",
    "Adversary<1, 2, 2>": "simple_adversary", "Adversary<1, 3, 3>": "simple_adversary_n4", "Push<1, 1, 2>": "simple_push",
    "SpeakerListener": "simple_speaker_listener", "Reference": "simple_reference", "Crypto": "simple_crypto",
}


def load_golden(tag):
    return dict(np.load(os.path.join(GOLDEN, tag + ".npz")))


def make_product_env(tag, **kw):
    from multiagent_particle_envs_b200 import make_env
    name, skw = CONFIGS[tag] if tag in CONFIGS else VARIANTS[tag]
    kw.update(skw)
    return make_env(name, benchmark=(name not in NO_BENCHMARK), **kw)


def descriptor(tag):
    from multiagent_particle_envs_b200 import scenarios
    name, kw = CONFIGS[tag] if tag in CONFIGS else VARIANTS[tag]
    return scenarios.load(name).Scenario(**kw).make_world().descriptor()


def step_flags(tag_or_golden):
    from multiagent_particle_envs_b200 import _lib
    g = load_golden(tag_or_golden) if isinstance(tag_or_golden, str) else tag_or_golden
    f = 0
    if int(g["prop_shared_reward"]):
        f |= _lib.FLAG_SHARED_REWARD
    if int(g["force_discrete"]):
        f |= _lib.FLAG_FORCE_DISCRETE_ACTION
    return f


def random_states(desc, n, rng, mode="mixed"):
    """seeded synthetic worlds in the oracle layout: reset-like, squeezed (contacts), fast/outside"""
    A, L, C = desc.n_agents, desc.n_landmarks, desc.dim_c
    pv = np.zeros((n, A, 4))
    pv[:, :, 0:2] = rng.uniform(-1, 1, (n, A, 2))
    lm = rng.uniform(-0.9, 0.9, (n, L, 2))
    kind = rng.randint(0, 4, n) if mode == "mixed" else np.zeros(n, int)
    sq = kind == 1
    pv[sq, :, 0:2] *= 0.3
    lm[sq] *= 0.3
    fast = kind == 2
    pv[fast, :, 0:2] *= 1.25
    pv[fast, :, 2:4] = rng.uniform(-1.5, 1.5, (int(fast.sum()), A, 2))
    tight = kind == 3
    pv[tight, :, 0:2] = rng.uniform(-0.12, 0.12, (int(tight.sum()), A, 2))
    comm = np.zeros((n, A, C))
    for i in range(A):
        if not desc.agent_silent[i]:
            comm[:, i, :] = rng.uniform(0, 1, (n, C)) * (rng.uniform(0, 1, (n, 1)) > 0.1)
        if not desc.agent_movable[i]:
            pv[:, i, 2:4] = 0.0
    return pv, lm, comm


def random_goals(n_goals, n_landmarks, n, rng):
    return rng.randint(0, max(n_landmarks, 1), (n, n_goals)).astype(np.int32)


def random_actions(act_dims, n, rng, temperature=2.0, movable=None):
    """probability vectors as MADDPG emits (softmax of logits) + uniform comm"""
    parts = []
    for i, d in enumerate(act_dims):
        mov = True if movable is None else bool(movable[i])
        if mov:
            logits = temperature * rng.randn(n, 5)
            p = np.exp(logits - logits.max(axis=1, keepdims=True))
            p /= p.sum(axis=1, keepdims=True)
            parts.append(p)
            d -= 5
        if d > 0:
            parts.append(rng.uniform(0, 1, (n, d)) * (rng.uniform(0, 1, (n, 1)) > 0.1))
    return np.concatenate(parts, axis=1)


# ---- launch shapes: which block size the library picks for a batch ----------------------------------
# Mirrors of the launch-shape rules in multiagent_particle_envs_b200/csrc/mpe_kernels.cu (sms = the device's SM count):
#   "step"   launch() -> launch_grid: the fused step runs whole 32-world tiles on the HOT kernel -- 1 warp per
#            block up to 16*sms tiles, 2 up to 64*sms, else 4 -- and the ragged tail (< 32 worlds) on the general kernel
#            at begin = whole tiles, in one 1-warp block (launch()).  Above 16*sms tiles the programs with a
#            hot_dense_fn take that 80-register build instead of hot_fn (launch()); make_program builds it
#            where kLowRegVariant holds: tag with 3 to 6 agents and spread N=4 (csrc/mpe_scenarios.cuh ~l.96, ~l.173).
#   "rollout" mpe_rollout: 1 warp per block up to 4*sms warps, 2 up to 64*sms, else 4
#   "policy"  mpe_rollout_policy: 1 up to 16*sms warps, 2 up to 64*sms, else 4
#   "mlp"     rollout_policy_mlp, all six forms: ceil(warps / sms) warps per block, capped at mlp_block_warps
#            (mirrored by mlp_programs.mlp_block_cap)
# The shared-memory caps (max_warps_per_block) never bind for the built-in scenarios at 4 warps per block.
STEP_DENSE_TAGS = ("simple_tag", "simple_tag_2v1", "simple_tag_4v2", "simple_spread_n4")   # the tags with a hot_dense_fn


def device_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def launch_shape(kernel, n, sms, cap=16):
    """(warps per block, #blocks, last block partial, worlds in the last warp) the library picks for n worlds.  For
    "step" this describes the HOT launch over the whole tiles; the tail is n % 32 worlds on the general kernel."""
    warps = n // 32 if kernel == "step" else (n + 31) // 32
    if kernel == "step":
        wpb = 1 if warps <= 16 * sms else (2 if warps <= 64 * sms else 4)
    elif kernel == "rollout":
        wpb = 1 if warps <= 4 * sms else (2 if warps <= 64 * sms else 4)
    elif kernel == "policy":
        wpb = 1 if warps <= 16 * sms else (2 if warps <= 64 * sms else 4)
    elif kernel == "mlp":
        wpb = max(1, min(cap, -(-warps // sms)))
    else:
        raise ValueError(kernel)
    blocks = -(-warps // wpb)
    last_rows = n % 32 if kernel == "step" else (n - 32 * (warps - 1))
    return wpb, blocks, warps % wpb != 0, last_rows if last_rows else 32


def step_uses_dense(tag, n, sms):
    return tag in STEP_DENSE_TAGS and n // 32 > 16 * sms


def regime_size(kernel, sms, wpb, cap=16, base=None):
    """A batch size for which `kernel` launches blocks of `wpb` warps with a partial last block (when wpb > 1) and a
    ragged last warp (17 worlds).  `base` (worlds) asks for a size just above it in that regime, e.g. 65 536 worlds
    plus a ragged tail."""
    if kernel == "mlp":
        lo = (wpb - 1) * sms + 1                 # ceil(warps / sms) == wpb from here on (up to wpb * sms, or the cap)
    else:
        lo = {1: 1, 2: {"rollout": 4, "policy": 16, "step": 16}[kernel] * sms + 1, 4: 64 * sms + 1}[wpb]
    warps = max(lo, base // 32 + 1 if base else lo)   # "step": whole tiles; otherwise warps including the ragged one
    while wpb > 1 and warps % wpb == 0:
        warps += 1
    n = warps * 32 + 17 if kernel == "step" else (warps - 1) * 32 + 17
    shape = launch_shape(kernel, n, sms, cap)
    assert shape[0] == wpb and shape[2] == (wpb > 1) and shape[3] == 17, (kernel, sms, wpb, n, shape)
    return n


def split_cols(a, dims):
    out, c = [], 0
    for d in dims:
        out.append(a[..., c:c + d])
        c += d
    return out


# ---- conditioning of the post-step velocity ---------------------------------------------------------
# integrate_state (core.py:158-169) makes each velocity component the sum v (1 - damping) + (u + sum of contact forces)
# dt / m.  In a squeezed world those forces are large and cancel, so the result can be small next to its terms; any
# fp32 evaluation then errs by a few ulps of the TERMS, which the per-element rtol of the small result does not cover.
VELOCITY_TERM_ULPS = 8


def velocity_term_scale(desc, pv0, lm, act, act_dims):
    """[n, A, 2]: per velocity component, the sum of |terms| of that sum (fp64, from the pre-step state and actions)"""
    A, L = desc.n_agents, desc.n_landmarks
    pos = np.concatenate([np.asarray(pv0, np.float64)[:, :, 0:2], np.asarray(lm, np.float64).reshape(len(pv0), L, 2)], 1)
    size = [desc.agent_size[i] for i in range(A)] + [desc.landmark_size[l] for l in range(L)]
    collide = [bool(desc.agent_collide[i]) for i in range(A)] + [bool(desc.landmark_collide[l]) for l in range(L)]
    F = np.zeros((len(pv0), A, 2))
    off = 0
    for i in range(A):
        if desc.agent_movable[i]:                                   # |u| (environment.py:174-181)
            a = np.asarray(act[:, off:off + 5], np.float64)
            F[:, i, 0] += np.abs(a[:, 1] - a[:, 2]) * desc.agent_sens[i]
            F[:, i, 1] += np.abs(a[:, 3] - a[:, 4]) * desc.agent_sens[i]
        off += act_dims[i]
    k = desc.contact_margin
    for a in range(A + L):                                          # |collision forces| (core.py:181-193)
        for b in range(a + 1, A + L):
            if not (collide[a] and collide[b]) or (a >= A and b >= A):
                continue
            delta = pos[:, a] - pos[:, b]
            dist = np.sqrt((delta ** 2).sum(-1, keepdims=True))
            pen = np.logaddexp(0, -(dist - size[a] - size[b]) / k) * k
            f = np.abs(desc.contact_force * delta / np.maximum(dist, 1e-30) * pen)
            for e in (a, b):
                if e < A:
                    F[:, e] += f
    mass = np.array([desc.agent_mass[i] for i in range(A)])[None, :, None]
    return np.abs(np.asarray(pv0, np.float64)[:, :, 2:4]) * (1 - desc.damping) + F / mass * desc.dt


# ---- accounting for contact-indicator mismatches between fp32 and fp64 ---------------------------------
# Rewards / benchmark_data contain indicator terms ([dist < size_a + size_b], [min dist < 0.1]).  An fp32
# evaluation may legitimately flip one when the fp64 distance sits within rounding of its threshold.  Every
# mismatch must be explained that way: (1) the difference is an integer multiple of the scenario's contact
# quantum and (2) some entity pair of that world is within `margin` of a threshold in the fp64 reference state.
CONTACT_QUANTUM = {"simple_spread": 1.0, "simple_tag": 10.0, "simple_world_comm": 1.0}   # world_comm: 5a + 2b
INFO_QUANTUM = 1.0                                                                       # counts


def scenario_of(tag):
    for name in ("simple_spread", "simple_tag", "simple_world_comm"):
        if tag.startswith(name):
            return name
    return tag


def threshold_margin(scn, pv_post, lm, a_size, l_size):
    """per world: min over entity pairs of |dist - threshold| in the given (fp64) post-step state"""
    p = np.asarray(pv_post, dtype=np.float64)[:, :, 0:2]
    lm = np.asarray(lm, dtype=np.float64)
    n, A = p.shape[:2]
    best = np.full(n, np.inf)
    for i in range(A):
        for j in range(i + 1, A):
            d = np.sqrt(((p[:, i] - p[:, j]) ** 2).sum(-1))
            best = np.minimum(best, np.abs(d - (a_size[i] + a_size[j])))
        for l in range(lm.shape[1]):
            d = np.sqrt(((p[:, i] - lm[:, l]) ** 2).sum(-1))
            best = np.minimum(best, np.abs(d - (a_size[i] + l_size[l])))
            if scn == "simple_spread":
                best = np.minimum(best, np.abs(d - 0.1))      # occupied_landmarks (simple_spread.py:56-57)
    return best


def explain_flag_mismatches(tag, rew, ref_rew, info, ref_info, pv_post64, lm64, a_size, l_size,
                            rtol=1e-5, atol=5e-6, margin=2e-6):
    """assert that every reward / info mismatch is a flipped contact indicator; returns #worlds with one"""
    scn = scenario_of(tag)
    ok = np.isclose(rew, ref_rew, rtol=rtol, atol=atol)
    bad = ~ok.all(axis=1)
    oki = None
    if info is not None and info.size:
        oki = np.isclose(info, ref_info, rtol=rtol, atol=atol)
        bad |= ~oki.reshape(oki.shape[0], -1).all(axis=1)
    if not bad.any():
        return 0
    q = CONTACT_QUANTUM.get(scn)
    assert q is not None, "%s has no contact indicators: reward mismatch in worlds %s" % (tag, np.where(bad)[0][:8])
    m = threshold_margin(scn, pv_post64, lm64, a_size, l_size)
    assert (m[bad] < margin).all(), "unexplained mismatch: worlds %s have no pair within %g of a threshold (margins %s)" % (
        np.where(bad)[0][:8], margin, m[bad][:8])
    d = (np.asarray(rew, np.float64) - ref_rew)[~ok] / q
    assert (np.abs(d - np.round(d)) < 1e-3).all() and (np.round(d) != 0).all(), "reward difference is not a multiple of %g: %s" % (q, d[:8])
    if oki is not None:
        di = (np.asarray(info, np.float64) - ref_info)[~oki]
        # counts differ by integers; simple_spread's info[0] is the reward itself (quantum 1 as well)
        assert (np.abs(di - np.round(di)) < 1e-3).all(), di[:8]
    return int(bad.sum())
