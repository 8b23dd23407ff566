"""CPU checks of IPPO's local critics (env.rollout_policy(..., critic=..., centralized_critic=False)): the fold on one
agent's observation and the float64 recipe models without rounding against the unfolded modules, every refusal
rollout_policy raises before the world is bound, the three C entry points and their device-less return codes, and the
launch bounds and programs of the new kernels against the mirrored tables."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from critic_helpers import CriticModel, make_critic, module_values
from helpers import TYPE_TAGS, make_product_env
from ippo_helpers import (LOCAL_PROGRAMS, RLOCAL_PROGRAMS, RLOCAL_WARPS, local_critic_block_cap,
                          local_critic_smem_warps, make_rcritic, min_count)
from mappo_helpers import FEATURE_NORM, TANH, make_mappo_actors
from mlp_programs import PROGRAMS
from rcritic_helpers import H, RecurrentModel
from rmappo_helpers import make_rmappo_actor, module_step
from test_cpu_mlp_block_table import max_threads_per_kernel

torch = pytest.importorskip("torch")
nn = torch.nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBS, ACT = [18] * 3, [5] * 3            # simple_spread N=3


@pytest.mark.parametrize("tanh", [False, True])
@pytest.mark.parametrize("fn", [False, True])
def test_the_local_fold_and_the_unrounded_model_equal_the_module(tanh, fn):
    """the critic folded on [obs_dim] (mappo_actor_params), evaluated by the centralized critic's recipe on [obs_k]
    without rounding, against the module in float64"""
    from multiagent_particle_envs_b200.environment import mappo_actor_params
    critic = make_critic([18], tanh, fn, device="cpu", eps=1e-3)
    params, got_tanh, got_fn, eps = mappo_actor_params([critic], [18], [1])
    assert (got_tanh, got_fn, eps) == (tanh, fn, 1e-3)
    assert [tuple(t.shape) for t in params[0]] == [(H, 18), (H,), (H, H), (H,), (1, H), (1,)]
    x = np.random.RandomState(0).randn(512, 18) * 2.0
    model = CriticModel([t.numpy() for t in params[0]], ((FEATURE_NORM if fn else 0) | (TANH if tanh else 0), eps), [18])
    model.t = [p.numpy() for p in params[0][0::2]]
    model.b = [p.numpy() for p in params[0][1::2]]
    x2 = model.hidden(model.hidden(model.input(x)[0], 0)[0], 1)[0]
    np.testing.assert_allclose(model.logits(x2)[:, 0], module_values(critic, x), rtol=0, atol=1e-10)


@pytest.mark.parametrize("tanh", [False, True])
@pytest.mark.parametrize("fn", [False, True])
def test_the_recurrent_local_fold_and_the_unrounded_model_equal_the_modules(tanh, fn):
    """rmappo_critic_params(critic, [obs_dim]) and RecurrentModel without rounding against the modules on obs_k"""
    from multiagent_particle_envs_b200.environment import rmappo_critic_params
    critic = make_rcritic([18], tanh, fn, device="cpu", eps=1e-3)
    params, got_tanh, got_fn, eps = rmappo_critic_params(critic, [18])
    assert (got_tanh, got_fn, eps) == (tanh, fn, 1e-3) and tuple(params[0].shape) == (H, 18)
    rng = np.random.RandomState(1)
    x, h = rng.randn(512, 18) * 2.0, np.tanh(rng.randn(512, H))
    net = ((FEATURE_NORM if fn else 0) | (TANH if tanh else 0), eps)
    v, hn = RecurrentModel([t.numpy() for t in params], net, tf32=False).step(x, h)
    v64, hn64 = module_step(critic, x, h)
    np.testing.assert_allclose(hn, hn64, rtol=0, atol=1e-10)
    np.testing.assert_allclose(v, v64, rtol=0, atol=1e-10)


def _seq(obs_dim, **kw):
    return make_critic([obs_dim], False, True, device="cpu", **kw)


def test_refusals_before_the_world_is_bound():
    """every ValueError and NotImplementedError of centralized_critic=False, raised before bind() (this machine has no
    device to bind to, so a refusal raised later would be a RuntimeError)"""
    env = make_product_env("simple_spread_n3", num_envs=64)
    mappo = make_mappo_actors(OBS, ACT, False, True, device="cpu")
    ractor = make_rmappo_actor(18, 5, False, True, device="cpu")
    kw = dict(action_mode="categorical", centralized_critic=False)
    cases = [
        (mappo, None, {}, ValueError, "needs a critic"),
        (mappo, _seq(54), {}, ValueError, "expected Linear weights"),                 # share_obs's width, not obs_dim
        (mappo, [_seq(18), _seq(18, seed=2), _seq(17)], {}, ValueError, "expected Linear weights"),
        (mappo, make_critic([18], True, True, device="cpu"), {}, ValueError, "activation"),
        (mappo, _seq(18, eps=1e-3), {}, ValueError, "eps"),
        (mappo, [_seq(18)] * 2, {}, ValueError, "list of 1 or 3"),
        ([ractor] * 3, make_rcritic([54], False, True, device="cpu"), {}, ValueError, "expected Linear weights"),
        ([ractor] * 3, make_rcritic([18], False, True, device="cpu"),
         dict(critic_rnn_states=torch.zeros(64, H)), ValueError, "critic_rnn_states"),
        ([ractor] * 3, make_rcritic([18], False, True, device="cpu"),
         dict(critic_rnn_states=torch.zeros(3, 64, H, dtype=torch.float64)), ValueError, "critic_rnn_states"),
        ([ractor] * 3, [make_rcritic([18], False, True, device="cpu", seed=s) for s in range(3)], {},
         NotImplementedError, "distinct"),
        ([nn.Sequential(nn.Linear(18, 64), nn.ReLU(), nn.Linear(64, 64), nn.ReLU(), nn.Linear(64, 5))] * 3, _seq(18),
         {}, NotImplementedError, "critic"),
    ]
    for actors, critic, extra, exc, match in cases:
        with pytest.raises(exc, match=match):
            env.rollout_policy(actors, 4, critic=critic, **kw, **extra)
    # a shared critic needs agents that observe alike
    tag = make_product_env("simple_tag", num_envs=64)
    shapes = tag.world.native_shapes()
    pols = make_mappo_actors(shapes.obs_dims, shapes.act_dims, False, True, device="cpu")
    with pytest.raises(ValueError, match="equal obs_dims"):
        tag.rollout_policy(pols, 4, critic=_seq(shapes.obs_dims[0]), **kw)
    assert env.world._native is None and tag.world._native is None


def test_local_critics_with_the_separated_runner_are_refused():
    env = make_product_env("simple_speaker_listener", num_envs=64)
    shapes = env.world.native_shapes()
    actors = [make_rmappo_actor(od, ad, False, True, device="cpu", seed=i)
              for i, (od, ad) in enumerate(zip(shapes.obs_dims, shapes.act_dims))]
    critics = [make_rcritic([od], False, True, device="cpu", seed=i) for i, od in enumerate(shapes.obs_dims)]
    with pytest.raises(NotImplementedError, match="separated"):
        env.rollout_policy(actors, 4, action_mode="categorical", critic=critics, centralized_critic=False)


# ---- the C ABI ----------------------------------------------------------------------------------------------------------
ENTRY_POINTS = {"mpe_rollout_policy_mappo_local_critic": "mpe_rollout_policy_mappo_critic",
                "mpe_rollout_policy_mappo_local_critic_episodes": "mpe_rollout_policy_mappo_critic_episodes",
                "mpe_critic_gru_local": "mpe_critic_gru"}
BAD_ARG, NO_DEVICE = -1, -5


def test_entry_points_are_declared_exported_and_bound_with_the_centralized_signatures():
    from multiagent_particle_envs_b200 import _lib
    header = open(os.path.join(ROOT, "include", "mpe_b200.h")).read()
    declared = set(re.findall(r"MPE_API[^;(]*?\b(mpe_[a-z_]+)\s*\(", header))
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name, base in ENTRY_POINTS.items():
        assert name in declared and name in _lib.EXPORTED_SYMBOLS and hasattr(lib, name), name
        assert _lib._SIGNATURES[name] == _lib._SIGNATURES[base], name
    assert _lib.MPE_ABI_VERSION == 1 and len(declared) == 44


def test_return_codes_without_a_device_are_the_centralized_ones():
    """every probe of the test files of the centralized critics, on both entry points of each pair"""
    import test_cpu_mappo_critic as mc
    import test_cpu_rmappo_critic as rc
    from multiagent_particle_envs_b200 import _lib
    shapes = make_product_env("simple_spread_n3", num_envs=64).world.native_shapes()   # device-less handle
    for name in ("mpe_rollout_policy_mappo_local_critic", "mpe_rollout_policy_mappo_local_critic_episodes"):
        probes = [dict(handle=None), dict(handle=shapes.handle, steps=-1), dict(handle=shapes.handle, weights=False),
                  dict(handle=shapes.handle), dict(handle=shapes.handle, count=3)]
        got = [mc._call(name, **kw) for kw in probes]
        assert got == [mc._call(ENTRY_POINTS[name], **kw) for kw in probes], name
        episodes = name.endswith("_episodes")
        assert got == [BAD_ARG, NO_DEVICE if episodes else BAD_ARG, NO_DEVICE if episodes else BAD_ARG, NO_DEVICE,
                       NO_DEVICE], name
    lib = _lib.load()
    per_agent = _lib.ptr_array([256] * _lib.MPE_MAX_AGENTS)

    def call(fn, handle, steps=4, episode_length=0, weights=True):
        w = [256 if weights else None] * 10
        return fn(handle, per_agent, per_agent, steps, episode_length, *w, 256, None, 256, 256, 0, 0.0, None)

    probes = [dict(handle=None), dict(handle=shapes.handle, steps=-1), dict(handle=shapes.handle, weights=False),
              dict(handle=shapes.handle, episode_length=3), dict(handle=shapes.handle)]
    got = [call(lib.mpe_critic_gru_local, **kw) for kw in probes]
    assert got == [call(lib.mpe_critic_gru, **kw) for kw in probes] == [rc._call(**kw) for kw in probes]
    assert got == [BAD_ARG, BAD_ARG, NO_DEVICE, NO_DEVICE, NO_DEVICE]


def _launch_bounds(pattern):
    from multiagent_particle_envs_b200 import _lib
    threads = max_threads_per_kernel(_lib.LIB_PATH)
    names = list(threads)
    demangled = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True,
                               check=True).stdout.split("\n")
    seen = {}
    for mangled, nm in zip(names, demangled):
        m = re.match(pattern, nm)
        if m:
            seen[(TYPE_TAGS[m.group(2)], bool(m.group(1)))] = threads[mangled]
    return seen


def test_launch_bounds_and_programs_are_the_mirrored_tables():
    """the MLP kernels: the programs whose smallest set fits, each at local_critic_block_cap warps; the recurrent one:
    the recurrent actor's programs at 8 warps"""
    seen = _launch_bounds(r"void mpe::mpe_policy_mappo_local_critic(_episode)?_kernel<mpe::(.+?)\s*>\(")
    assert {t for t, _ in seen} == set(LOCAL_PROGRAMS) and len(seen) == 2 * len(LOCAL_PROGRAMS) == 30
    for (tag, episodes), got in seen.items():
        assert got == 32 * local_critic_block_cap(tag, episodes), (tag, episodes, got)
    seen = _launch_bounds(r"void mpe::mpe_critic_gru_local_kernel()<mpe::(.+?)\s*>\(")
    assert {t for t, _ in seen} == set(RLOCAL_PROGRAMS) and set(seen.values()) == {32 * RLOCAL_WARPS}


def test_the_fit_rule():
    """the figures the kernels' static_asserts state"""
    assert set(PROGRAMS) - set(LOCAL_PROGRAMS) == {"simple_tag_4v2", "simple_tag_6v2"}
    assert local_critic_smem_warps("simple_spread_n3", 3) == 23 and local_critic_smem_warps("simple_spread_n6", 1) == 4
    assert local_critic_smem_warps("simple_spread_n4", 4) == 7
    assert local_critic_smem_warps("simple_spread_n5", 5) < 1 and local_critic_smem_warps("simple_spread_n6", 6) < 1
    assert min_count("simple_tag") == 4 and min_count("simple_spread_n6") == 1
