"""CPU checks of MAPPO's centralized critic in the in-kernel rollout (mpe_rollout_policy_mappo_critic[_episodes]): its
fold and the float64 recipe model without rounding against the unfolded module, the critics mappo_critic_params and
rollout_policy refuse, the C ABI and its device-less return codes, and the launch bounds of the 30 kernels against the
mirrored block table."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from critic_helpers import (CRITIC_PROGRAMS, H, CriticModel, critic_block_cap, critic_smem_warps, make_critic,
                            module_values)
from helpers import TYPE_TAGS, make_product_env
from mappo_helpers import FEATURE_NORM, TANH, make_mappo_actors
from mlp_programs import shapes_of
from test_cpu_mlp_block_table import max_threads_per_kernel

torch = pytest.importorskip("torch")
nn = torch.nn

ROOT = os.path.dirname(os.path.abspath(__file__))
OBS, ACT = [18] * 3, [5] * 3            # simple_spread N=3: D = 54


def _params(critic, obs=OBS):
    from multiagent_particle_envs_b200.environment import mappo_critic_params
    return mappo_critic_params(critic, obs)


@pytest.mark.parametrize("tanh", [False, True])
@pytest.mark.parametrize("fn", [False, True])
def test_the_fold_and_the_unrounded_model_equal_the_module(tanh, fn):
    """the folded float64 critic, evaluated by the recipe without rounding, against the module in float64"""
    critic = make_critic(OBS, tanh, fn, device="cpu", eps=1e-3)
    params, got_tanh, got_fn, eps = _params(critic)
    assert (got_tanh, got_fn, eps) == (tanh, fn, 1e-3) and len(params) == 1
    assert [tuple(t.shape) for t in params[0]] == [(H, 54), (H,), (H, H), (H,), (1, H), (1,)]
    assert all(t.dtype == torch.float64 for t in params[0])
    rng = np.random.RandomState(0)
    x = rng.randn(512, 54) * 2.0
    model = CriticModel([t.numpy() for t in params[0]], ((FEATURE_NORM if fn else 0) | (TANH if tanh else 0), eps), OBS)
    # the recipe with every rounding off: float64 weights, no TF32
    model.t = [p.numpy() for p in params[0][0::2]]
    model.b = [p.numpy() for p in params[0][1::2]]
    x0 = model.input(x)[0]
    x1 = model.hidden(x0, 0)[0]
    x2 = model.hidden(x1, 1)[0]
    np.testing.assert_allclose(model.logits(x2)[:, 0], module_values(critic, x), rtol=0, atol=1e-10)


def test_the_rounded_model_is_near_the_module():
    critic = make_critic(OBS, True, True, device="cpu")
    params, tanh, fn, eps = _params(critic)
    x = np.random.RandomState(1).randn(256, 54)
    v, bound = CriticModel([t.numpy() for t in params[0]], (FEATURE_NORM | TANH, eps), OBS).values(x)
    d = np.abs(v - module_values(critic, x))
    assert 0 < d.max() < 5e-2 and (bound > 0).all()


def test_shared_and_per_agent_lists():
    """one module, [critic] * n and [critic] are one shared critic; n distinct modules are n critics"""
    a = make_critic(OBS, False, True, device="cpu", seed=1)
    b = make_critic(OBS, False, True, device="cpu", seed=2)
    assert len(_params(a)[0]) == 1 and len(_params([a] * 3)[0]) == 1 and len(_params([a])[0]) == 1
    assert len(_params([a, b, a])[0]) == 3


def _with(i, m, base=None):
    base = base if base is not None else make_critic(OBS, False, True, device="cpu")
    return nn.Sequential(*[m if j == i else x for j, x in enumerate(base)])


@pytest.mark.parametrize("critic,match", [
    (_with(1, nn.Linear(53, 64)), "expected Linear weights"),                     # input width other than D
    (_with(0, nn.LayerNorm(53)), "expected Linear weights"),
    (_with(1, nn.Linear(54, 64, bias=False)), "bias"),
    (_with(7, nn.Linear(64, 1, bias=False)), "bias"),
    (_with(7, nn.Linear(64, 2)), "expected Linear weights"),                      # not one output
    (_with(4, nn.ReLU()), "must be"),                                             # wrong layer list
    (nn.Sequential(*list(make_critic(OBS, False, True, device="cpu"))[:-1]), "must be"),
    (_with(3, nn.LayerNorm(64, elementwise_affine=False)), "elementwise_affine"),
    (_with(3, nn.LayerNorm(64, eps=1e-3)), "same eps"),
    (_with(2, nn.Tanh()), "must be"),                                             # mixed activations
    ((nn.Linear(54, 1),), "must be"),
    ([make_critic(OBS, False, True, device="cpu")] * 2, "list of 1 or 3"),        # list length other than 1 or n
    ("critic", "one module"),
])
def test_refuses_malformed_critics(critic, match):
    with pytest.raises(ValueError, match=match):
        _params(critic)


def test_refusals_without_a_device():
    """a critic with any actor but MAPPO's MLP actor, or with the softmax mode, is refused before the env is bound"""
    from rmappo_helpers import make_rmappo_actor
    env = make_product_env("simple_spread_n3", num_envs=64)
    critic = make_critic(OBS, False, True, device="cpu")
    mappo = make_mappo_actors(OBS, ACT, False, True, device="cpu")
    maddpg = [nn.Sequential(nn.Linear(18, 64), nn.ReLU(), nn.Linear(64, 64), nn.ReLU(), nn.Linear(64, 5))] * 3
    one_layer = [nn.Sequential(nn.Linear(18, 64), nn.ReLU(), nn.Linear(64, 5))] * 3
    gru = [make_rmappo_actor(18, 5, False, True, device="cpu")] * 3
    for actors in (maddpg, one_layer, gru):
        with pytest.raises(NotImplementedError, match="critic"):
            env.rollout_policy(actors, 4, action_mode="categorical", critic=critic)
    with pytest.raises(NotImplementedError, match="critic"):
        env.rollout_policy(mappo, 4, critic=critic)


# ---- the C ABI ----------------------------------------------------------------------------------------------------------
ENTRY_POINTS = ("mpe_rollout_policy_mappo_critic", "mpe_rollout_policy_mappo_critic_episodes")
BAD_ARG, NO_DEVICE = -1, -5


def test_entry_points_are_declared_exported_and_bound():
    from multiagent_particle_envs_b200 import _lib
    header = open(os.path.join(os.path.dirname(ROOT), "include", "mpe_b200.h")).read()
    declared = set(re.findall(r"MPE_API[^;(]*?\b(mpe_[a-z_]+)\s*\(", header))
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name, base in zip(ENTRY_POINTS, ("mpe_rollout_policy_mappo", "mpe_rollout_policy_mappo_episodes")):
        assert name in declared and name in _lib.EXPORTED_SYMBOLS and hasattr(lib, name), name
        # MAPPO's parameters with (critic_count, six pointer arrays, values, final_values) after (net_flags, ln_eps)
        got, want = _lib._SIGNATURES[name][1], list(_lib._SIGNATURES[base][1])
        assert got == want[:-3] + [ctypes.c_int32] + [_lib._PP] * 6 + [_lib._P, _lib._P] + want[-3:], name
    assert _lib.MPE_ABI_VERSION == 1


def _call(name, handle, steps=4, weights=True, count=1):
    """`name` (a critic entry point, or MAPPO's) with aligned dummy pointers (every probe returns before one is used)"""
    from multiagent_particle_envs_b200 import _lib
    lib = _lib.load()
    argtypes = _lib._SIGNATURES[name][1]
    per_agent = _lib.ptr_array([256] * _lib.MPE_MAX_AGENTS)
    args = [256 if t is _lib._P else per_agent if t is _lib._PP else 1 if t.__name__ == "c_int" else 0 for t in argtypes]
    args[0], args[-1] = handle, None
    args[5:11] = [per_agent if weights else None] * 6
    args[11], args[12] = 64, steps
    if "critic" in name:
        args[-12] = count
    return getattr(lib, name)(*args)


def test_entry_point_return_codes_without_a_device():
    """equal to MAPPO's: the single-episode form refuses a negative n_steps and null weight arrays before it asks for
    the device, the episode form asks for the device first"""
    shapes = make_product_env("simple_spread_n3", num_envs=64).world.native_shapes()   # device-less handle
    for name, base in zip(ENTRY_POINTS, ("mpe_rollout_policy_mappo", "mpe_rollout_policy_mappo_episodes")):
        episodes = name.endswith("_episodes")
        probes = [dict(handle=None), dict(handle=shapes.handle, steps=-1), dict(handle=shapes.handle, weights=False),
                  dict(handle=shapes.handle)]
        want = [BAD_ARG, NO_DEVICE if episodes else BAD_ARG, NO_DEVICE if episodes else BAD_ARG, NO_DEVICE]
        assert [_call(name, **kw) for kw in probes] == want, name
        assert [_call(base, **kw) for kw in probes] == want, base
        assert _call(name, shapes.handle, count=2) == NO_DEVICE and _call(name, shapes.handle, count=3) == NO_DEVICE


def test_launch_bounds_are_the_mirrored_table():
    """the 30 kernels: 15 programs x (one episode, episodes), each at critic_block_cap warps"""
    from multiagent_particle_envs_b200 import _lib
    threads = max_threads_per_kernel(_lib.LIB_PATH)
    names = list(threads)
    demangled = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True,
                               check=True).stdout.split("\n")
    seen = {}
    for mangled, nm in zip(names, demangled):
        m = re.match(r"void mpe::mpe_policy_mappo_critic(_episode)?_kernel<mpe::(.+?)\s*>\(", nm)
        if m:
            seen[(TYPE_TAGS[m.group(2)], bool(m.group(1)))] = threads[mangled]
    assert {t for t, _ in seen} == set(CRITIC_PROGRAMS) and len(seen) == 30
    for (tag, episodes), got in seen.items():
        assert got == 32 * critic_block_cap(tag, episodes), (tag, episodes, got)


def test_the_shared_memory_figures():
    """the figures the kernel's static_asserts state: where one shared critic fits, and n per-agent ones"""
    assert critic_smem_warps("simple_spread_n3", 1) == 34 and critic_smem_warps("simple_spread_n3", 3) == 12
    assert critic_smem_warps("simple_spread_n5", 1) == 7 and critic_smem_warps("simple_tag_4v2", 1) == 6
    assert critic_smem_warps("simple_spread_n6", 1) < 1 and critic_smem_warps("simple_tag_6v2", 1) < 1
    fit = {t for t in CRITIC_PROGRAMS if critic_smem_warps(t, len(shapes_of(t)[0])) >= 1}
    assert fit == {"simple", "simple_spread_n2", "simple_spread_n3", "simple_tag_1v1", "simple_tag_2v1",
                   "simple_adversary", "simple_push", "simple_speaker_listener", "simple_reference", "simple_crypto"}
