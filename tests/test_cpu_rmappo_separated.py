"""CPU checks of rMAPPO's separated runner on simple_speaker_listener (per-agent recurrent actors and critics,
mpe_rollout_policy_gru_separated[_episodes], mpe_critic_gru_separated): the per-agent fold and the float64 recipe model
without rounding against each agent's modules, the refusals made before the world is bound, the C ABI and its
device-less return codes, the workspace and shared-memory sizes, and the launch bounds of the new kernels."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from helpers import TYPE_TAGS, make_product_env
from mappo_helpers import FEATURE_NORM, TANH
from rmappo_helpers import H, RecurrentModel, make_rmappo_actor, module_step
from test_cpu_mlp_block_table import max_threads_per_kernel

torch = pytest.importorskip("torch")
nn = torch.nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TAG = "simple_speaker_listener"
OBS, ACT = [3, 11], [3, 5]               # the speaker sees the goal colour and utters; the listener moves
WARPS = 8
SMEM_OPTIN_BYTES = 232448


def _agents(tanh=False, fn=True, eps=1e-5, seeds=(3, 4)):
    return [make_rmappo_actor(od, ad, tanh, fn, seed=s, eps=eps, device="cpu") for od, ad, s in zip(OBS, ACT, seeds)]


def _critics(tanh=False, fn=True, eps=1e-5, seeds=(5, 6)):
    return [make_rmappo_actor(sum(OBS), 1, tanh, fn, seed=s, eps=eps, device="cpu") for s in seeds]


def image_floats(obs_dim, act_dim):
    """GruAgentShape in csrc/mpe_kernels.cu: the TF32 B fragments of W1 (obs_dim rounded up to 8), W2, W_ih, W_hh (24
    n-tiles each) and W3 (act_dim rounded up to 8), then b1, b2, b_ih, b_hh, b3; padded to 16 bytes"""
    kt1, nout = (obs_dim + 7) // 8, (act_dim + 7) // 8 * 8
    return (64 * 8 * (kt1 + 8 + 2 * 24 + nout // 8) + 64 + 64 + 192 + 192 + nout + 3) & ~3


def warp_floats(obs_dims, act_dims):
    """MlpShape::kWarpFloats: the observation tile (odd row pitch) and the 32 x (max NOUT + 1) logit tile"""
    def pitch(od):
        unit = 2 if od % 2 == 0 else 1
        return ((od // unit) | 1) * unit
    obs_tile = (max(32 * pitch(od) for od in obs_dims) + 3) & ~3
    return (obs_tile + 32 * (max((ad + 7) // 8 * 8 for ad in act_dims) + 1) + 3) & ~3


def test_image_and_shared_memory_sizes():
    """the two images do not fit in shared memory together; one slot for the larger and 8 warps' tiles do"""
    speaker, listener = (4 * image_floats(od, ad) for od, ad in zip(OBS, ACT))
    assert (speaker, listener) == (120864, 122912)
    assert speaker + listener > SMEM_OPTIN_BYTES
    slot = 16 + max(speaker, listener) + WARPS * 4 * warp_floats(OBS, ACT)   # the mbarrier header, slot and tiles
    assert slot <= SMEM_OPTIN_BYTES
    shapes = make_product_env(TAG, num_envs=64).world.native_shapes()
    assert shapes.gru_separated_workspace_bytes() == speaker + listener


@pytest.mark.parametrize("tanh", [False, True])
@pytest.mark.parametrize("fn", [False, True])
def test_the_per_agent_fold_and_the_unrounded_model_equal_the_modules(tanh, fn):
    """each agent's tuple folded by rmappo_actor_params on its own sizes, evaluated without rounding, against its
    base -> gru -> norm -> head in float64"""
    from multiagent_particle_envs_b200.environment import rmappo_actor_params
    rng = np.random.RandomState(0)
    for actor, od, ad in zip(_agents(tanh, fn, eps=1e-3), OBS, ACT):
        params, got_tanh, got_fn, eps = rmappo_actor_params([actor], [od], [ad])
        assert (got_tanh, got_fn, eps) == (tanh, fn, 1e-3)
        assert [tuple(t.shape) for t in params] == [(64, od), (64,), (64, 64), (64,), (192, 64), (192,), (192, 64),
                                                    (192,), (ad, 64), (ad,)]
        obs, h = rng.randn(512, od) * 2.0, np.tanh(rng.randn(512, H))
        net = ((FEATURE_NORM if fn else 0) | (TANH if tanh else 0), eps)
        z, hn = RecurrentModel([t.numpy() for t in params], net, tf32=False).step(obs, h)
        z64, hn64 = module_step(actor, obs, h)
        np.testing.assert_allclose(hn, hn64, rtol=0, atol=1e-10)
        np.testing.assert_allclose(z, z64, rtol=0, atol=1e-10)


def test_the_existing_folds_still_refuse_distinct_tuples():
    from multiagent_particle_envs_b200.environment import rmappo_actor_params, rmappo_critic_params
    a, b = _agents()
    with pytest.raises(NotImplementedError, match="shared"):
        rmappo_actor_params([a, b], OBS, ACT)
    with pytest.raises(NotImplementedError, match="distinct"):
        rmappo_critic_params(_critics(), OBS)


def _refused(exc, match, **kw):
    env = make_product_env(TAG, num_envs=64)
    args = dict(policies=_agents(), n_steps=4, action_mode="categorical")
    args.update(kw)
    with pytest.raises(exc, match=match):
        env.rollout_policy(args.pop("policies"), args.pop("n_steps"), **args)
    assert env.world._native is None   # refused before the world is bound


def test_refusals_before_the_world_is_bound():
    speaker, listener = _agents()
    relu, tanh = _agents(False), _agents(True)
    _refused(ValueError, "agent 0's recurrent actor", policies=[listener, speaker])       # dims of the other agent
    _refused(ValueError, "agent 1's recurrent actor", policies=[speaker, speaker[:3] + (nn.Linear(64, 7),)])
    _refused(ValueError, "same activation", policies=[relu[0], tanh[1]])
    _refused(ValueError, "same activation", policies=[speaker, _agents(fn=False)[1]])
    _refused(ValueError, "same activation", policies=[speaker, _agents(eps=1e-3)[1]])
    _refused(ValueError, "list of 2 recurrent critics", critic=_critics()[0])             # one critic tuple
    _refused(ValueError, "list of 2 recurrent critics", critic=_critics() + _critics()[:1])
    _refused(ValueError, "critic must use the actors'", critic=_critics(tanh=True))
    _refused(ValueError, "recurrent critic must be", critic=[_critics()[0], _agents()[1]])   # a critic of the wrong width
    _refused(ValueError, "critic_rnn_states", critic=_critics(), critic_rnn_states=torch.zeros(64, 64))
    _refused(ValueError, "rnn_states", rnn_states=torch.zeros(64, 64))
    _refused(ValueError, "rnn_states", rnn_states=torch.zeros(2, 64, 64))                   # not on the env's device
    _refused(ValueError, "episode_length", episode_length=2, rnn_states=torch.zeros(2, 64, 64))
    _refused(ValueError, "episode_length", episode_length=2, critic=_critics(), critic_rnn_states=torch.zeros(2, 64, 64))
    _refused(NotImplementedError, "categorical", action_mode="softmax")
    seq = nn.Sequential(nn.Linear(sum(OBS), 64), nn.ReLU(), nn.LayerNorm(64), nn.Linear(64, 64), nn.ReLU(),
                        nn.LayerNorm(64), nn.Linear(64, 1))
    _refused(NotImplementedError, "pairs", critic=[seq, seq])                                  # the pairing rule


# ---- the C ABI ----------------------------------------------------------------------------------------------------------
ENTRY_POINTS = ("mpe_rollout_policy_gru_separated", "mpe_rollout_policy_gru_separated_episodes",
                "mpe_rollout_policy_gru_separated_workspace_bytes", "mpe_critic_gru_separated")
BAD_ARG, UNSUPPORTED, NO_DEVICE = -1, -3, -5


def test_entry_points_are_declared_exported_and_bound():
    from multiagent_particle_envs_b200 import _lib
    header = open(os.path.join(ROOT, "include", "mpe_b200.h")).read()
    declared = set(re.findall(r"MPE_API[^;(]*?\b(mpe_[a-z_]+)\s*\(", header))
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in ENTRY_POINTS:
        assert name in declared and name in _lib.EXPORTED_SYMBOLS and hasattr(lib, name), name
    sig = _lib._SIGNATURES
    for name, base in zip(ENTRY_POINTS[:2], ("mpe_rollout_policy_gru", "mpe_rollout_policy_gru_episodes")):
        # the shared actor's parameters with a pointer array per weight and (workspace, bytes) after the state records
        got, want = sig[name][1], list(sig[base][1])
        assert got == want[:5] + [_lib._PP] * 10 + want[15:-5] + [_lib._P, ctypes.c_int64] + want[-5:], name
    got, want = sig["mpe_critic_gru_separated"][1], sig["mpe_critic_gru"][1]
    assert got == want[:5] + [_lib._PP] * 10 + want[15:]
    assert sig["mpe_rollout_policy_gru_separated_workspace_bytes"] == (ctypes.c_int64, [_lib._P])
    assert _lib.MPE_ABI_VERSION == 1


def _call(name, handle, steps=4, weights=True):
    """`name` with aligned dummy pointers (every probe returns before one is used)"""
    from multiagent_particle_envs_b200 import _lib
    lib = _lib.load()
    argtypes = _lib._SIGNATURES[name][1]
    per_agent = _lib.ptr_array([256] * _lib.MPE_MAX_AGENTS)
    args = [256 if t is _lib._P else per_agent if t is _lib._PP else 1 if t.__name__ == "c_int" else 0 for t in argtypes]
    args[0], args[-1] = handle, None
    if name == "mpe_critic_gru_separated":
        args[3] = steps
        args[5:15] = [per_agent if weights else None] * 10
    else:
        args[5:15] = [per_agent if weights else None] * 10
        args[15], args[16] = 64, steps
        args[argtypes.index(ctypes.c_int64)] = 1 << 20
    return getattr(lib, name)(*args)


def test_entry_point_return_codes_without_a_device():
    """the rollouts as the shared actor's: the single-episode form refuses a negative n_steps and a null weight array
    before it asks for the device, the episode form asks first; the critics as mpe_critic_gru; the workspace size needs
    no device"""
    from multiagent_particle_envs_b200 import _lib
    shapes = make_product_env(TAG, num_envs=64).world.native_shapes()   # device-less handle
    for name in ENTRY_POINTS[:2]:
        episodes = name.endswith("_episodes")
        probes = [dict(handle=None), dict(handle=shapes.handle, steps=-1), dict(handle=shapes.handle, weights=False),
                  dict(handle=shapes.handle)]
        want = [BAD_ARG, NO_DEVICE if episodes else BAD_ARG, NO_DEVICE if episodes else BAD_ARG, NO_DEVICE]
        assert [_call(name, **kw) for kw in probes] == want, name
    name = "mpe_critic_gru_separated"
    probes = [dict(handle=None), dict(handle=shapes.handle, steps=-1), dict(handle=shapes.handle, weights=False),
              dict(handle=shapes.handle)]
    assert [_call(name, **kw) for kw in probes] == [BAD_ARG, BAD_ARG, NO_DEVICE, NO_DEVICE]
    lib = _lib.load()
    spread = make_product_env("simple_spread_n3", num_envs=64).world.native_shapes()
    assert lib.mpe_rollout_policy_gru_separated_workspace_bytes(None) == BAD_ARG
    assert lib.mpe_rollout_policy_gru_separated_workspace_bytes(spread.handle) == UNSUPPORTED
    assert lib.mpe_rollout_policy_gru_separated_workspace_bytes(shapes.handle) == 120864 + 122912
    with pytest.raises(_lib.MpeError, match="no compiled"):
        spread.require_gru_separated()
    shapes.require_gru_separated()


def test_launch_bounds_are_8_warps():
    """the image kernel and the three per-agent kernels, for speaker_listener only"""
    from multiagent_particle_envs_b200 import _lib
    threads = max_threads_per_kernel(_lib.LIB_PATH)
    names = list(threads)
    demangled = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True,
                               check=True).stdout.split("\n")
    seen = {}
    for mangled, nm in zip(names, demangled):
        m = re.match(r"void mpe::(mpe_policy_gru_separated(?:_episode)?_kernel|mpe_critic_gru_separated_kernel|"
                     r"mpe_gru_image_kernel)<mpe::(.+?)\s*>\(", nm)
        if m:
            seen[(m.group(1), TYPE_TAGS[m.group(2)])] = threads[mangled]
    assert seen == {("mpe_policy_gru_separated_kernel", TAG): 32 * WARPS,
                    ("mpe_policy_gru_separated_episode_kernel", TAG): 32 * WARPS,
                    ("mpe_critic_gru_separated_kernel", TAG): 32 * WARPS,
                    ("mpe_gru_image_kernel", TAG): 256}
