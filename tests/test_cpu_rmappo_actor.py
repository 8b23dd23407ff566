"""CPU checks of MAPPO's recurrent actor in the in-kernel rollout (mpe_rollout_policy_gru[_episodes]): the tuples
rmappo_actor_params accepts and refuses, its fold, the float64 recipe model without rounding against the unfolded
modules, the C ABI and its device-less return codes, and the launch bounds of the 14 kernels against the mirrored
block table."""
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
OBS, ACT = [18] * 3, [5] * 3            # simple_spread N=3
# the programs the recurrent actor is built for (GruBuilt) and its block size, both forms (gru_block_warps)
GRU_PROGRAMS = ("simple", "simple_spread_n2", "simple_spread_n3", "simple_spread_n4", "simple_spread_n5",
                "simple_spread_n6", "simple_reference")
GRU_WARPS = 8


def _params(actor=None, n=3, obs=OBS, act=ACT, pols=None):
    from multiagent_particle_envs_b200.environment import rmappo_actor_params
    return rmappo_actor_params(pols if pols is not None else [actor] * n, obs, act)


@pytest.mark.parametrize("tanh", [False, True])
@pytest.mark.parametrize("fn", [False, True])
def test_the_fold_and_the_unrounded_model_equal_the_modules(tanh, fn):
    """the folded float64 network (RecurrentModel without rounding) against base -> gru -> norm -> head in float64, on
    random observations and hidden states"""
    actor = make_rmappo_actor(18, 5, tanh, fn, device="cpu", eps=1e-3)
    params, got_tanh, got_fn, eps = _params(actor)
    assert (got_tanh, got_fn, eps) == (tanh, fn, 1e-3)
    assert [tuple(t.shape) for t in params] == [(64, 18), (64,), (64, 64), (64,), (192, 64), (192,), (192, 64), (192,),
                                                (5, 64), (5,)]
    assert all(t.dtype == torch.float64 for t in params)
    rng = np.random.RandomState(0)
    obs, h = rng.randn(512, 18) * 2.0, np.tanh(rng.randn(512, H))
    net = ((FEATURE_NORM if fn else 0) | (TANH if tanh else 0), eps)
    z, hn = RecurrentModel([t.numpy() for t in params], net, tf32=False).step(obs, h)
    z64, hn64 = module_step(actor, obs, h)
    np.testing.assert_allclose(hn, hn64, rtol=0, atol=1e-10)
    np.testing.assert_allclose(z, z64, rtol=0, atol=1e-10)


def test_the_rounded_model_is_near_the_modules():
    actor = make_rmappo_actor(18, 5, True, True, device="cpu")
    params, tanh, fn, eps = _params(actor)
    rng = np.random.RandomState(1)
    obs, h = rng.randn(256, 18), np.tanh(rng.randn(256, H))
    z, hn = RecurrentModel([t.numpy() for t in params], (FEATURE_NORM | TANH, eps)).step(obs, h)
    z64, hn64 = module_step(actor, obs, h)
    assert 0 < np.abs(hn - hn64).max() < 5e-2 and np.abs(z - z64).max() < 5e-2


def _variant(**kw):
    """a seeded actor with one part replaced"""
    base, gru, norm, head = make_rmappo_actor(18, 5, False, True, device="cpu")
    if "gru" in kw:
        gru = kw["gru"]
    if "norm" in kw:
        norm = kw["norm"]
    if "head" in kw:
        head = kw["head"]
    if "base" in kw:
        base = kw["base"](base)
    return (base, gru, norm, head)


def _swap(i, m):
    return lambda base: nn.Sequential(*[m if j == i else x for j, x in enumerate(base)])


@pytest.mark.parametrize("actor,match", [
    (_variant(gru=nn.GRU(64, 64, num_layers=2)), "num_layers=1"),
    (_variant(gru=nn.GRU(64, 64, bidirectional=True)), "num_layers=1"),
    (_variant(gru=nn.GRU(64, 64, bias=False)), "bias=True"),
    (_variant(gru=nn.GRU(64, 32)), "nn.GRU\\(64, 64\\)"),
    (_variant(gru=nn.GRU(32, 64)), "nn.GRU\\(64, 64\\)"),
    (_variant(gru=nn.LSTM(64, 64)), "nn.GRU"),
    (_variant(norm=nn.LayerNorm(64, elementwise_affine=False)), "elementwise_affine"),
    (_variant(norm=nn.LayerNorm(64, eps=1e-3)), "same eps"),
    (_variant(norm=nn.LayerNorm(32)), "LayerNorm\\(64\\)"),
    (_variant(norm=nn.Identity()), "LayerNorm\\(64\\)"),
    (_variant(head=nn.Linear(64, 7)), "head"),
    (_variant(head=nn.Linear(64, 5, bias=False)), "bias"),
    (_variant(base=_swap(2, nn.Tanh())), "base must be"),                        # mixed activations
    (_variant(base=_swap(3, nn.LayerNorm(64, elementwise_affine=False))), "elementwise_affine"),
    (_variant(base=_swap(3, nn.LayerNorm(64, eps=1e-3))), "same eps"),
    (_variant(base=_swap(1, nn.Linear(18, 32))), "expected Linear weights"),       # a hidden width other than 64
    (_variant(base=_swap(4, nn.Linear(64, 64, bias=False))), "bias"),
    (_variant(base=lambda b: nn.Sequential(*list(b)[:-1])), "base must be"),      # no last LayerNorm
    (_variant()[:3], "must be"),
])
def test_refuses_malformed_actors(actor, match):
    with pytest.raises(ValueError, match=match):
        _params(actor)


def test_distinct_tuples_are_not_shared():
    """one policy object for every agent (share_policy): equal values in distinct tuples are refused"""
    a = make_rmappo_actor(18, 5, False, True, device="cpu")
    _params(a)
    with pytest.raises(NotImplementedError, match="shared"):
        _params(pols=[a, tuple(list(a)), a])
    with pytest.raises(ValueError, match="same observation and action sizes"):
        _params(a, n=2, obs=[8, 10], act=[3, 5])


# ---- the C ABI ----------------------------------------------------------------------------------------------------------
ENTRY_POINTS = ("mpe_rollout_policy_gru", "mpe_rollout_policy_gru_episodes")
BAD_ARG, NO_DEVICE = -1, -5


def test_entry_points_are_declared_exported_and_bound():
    from multiagent_particle_envs_b200 import _lib
    header = open(os.path.join(ROOT, "include", "mpe_b200.h")).read()
    declared = set(re.findall(r"MPE_API[^;(]*?\b(mpe_[a-z_]+)\s*\(", header))
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name, base in zip(ENTRY_POINTS, ("mpe_rollout_policy_mappo", "mpe_rollout_policy_mappo_episodes")):
        assert name in declared and name in _lib.EXPORTED_SYMBOLS and hasattr(lib, name), name
        # MAPPO's parameters with ten single weight pointers for the six per-agent arrays and (rnn_state,
        # rnn_state_record) before (net_flags, ln_eps, done, flags, stream)
        got, want = _lib._SIGNATURES[name][1], list(_lib._SIGNATURES[base][1])
        assert got == want[:5] + [_lib._P] * 10 + want[11:-5] + [_lib._P, _lib._P] + want[-5:], name
    assert _lib.MPE_ABI_VERSION == 1


def _call(name, handle, steps=4, weights=True):
    """`name` with aligned dummy pointers (every probe returns before one is used)"""
    from multiagent_particle_envs_b200 import _lib
    lib = _lib.load()
    argtypes = _lib._SIGNATURES[name][1]
    per_agent = _lib.ptr_array([256] * _lib.MPE_MAX_AGENTS)
    args = [256 if t is _lib._P else per_agent if t is _lib._PP else 1 if t.__name__ == "c_int" else 0 for t in argtypes]
    args[0], args[-1] = handle, None
    args[5:15] = [256 if weights else None] * 10
    args[15], args[16] = 64, steps
    return getattr(lib, name)(*args)


def test_entry_point_return_codes_without_a_device():
    """as MAPPO's: the single-episode form refuses a negative n_steps and a null weight before it asks for the device,
    the episode form asks for the device first"""
    shapes = make_product_env("simple_spread_n3", num_envs=64).world.native_shapes()   # device-less handle
    for name in ENTRY_POINTS:
        episodes = name.endswith("_episodes")
        probes = [dict(handle=None), dict(handle=shapes.handle, steps=-1), dict(handle=shapes.handle, weights=False),
                  dict(handle=shapes.handle)]
        want = [BAD_ARG, NO_DEVICE if episodes else BAD_ARG, NO_DEVICE if episodes else BAD_ARG, NO_DEVICE]
        assert [_call(name, **kw) for kw in probes] == want, name


def test_launch_bounds_are_the_mirrored_table():
    """the 14 kernels: 7 programs x (one episode, episodes), every one at GRU_WARPS warps"""
    from multiagent_particle_envs_b200 import _lib
    threads = max_threads_per_kernel(_lib.LIB_PATH)
    names = list(threads)
    demangled = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True,
                               check=True).stdout.split("\n")
    seen = {}
    for mangled, nm in zip(names, demangled):
        m = re.match(r"void mpe::mpe_policy_gru(_episode)?_kernel<mpe::(.+?)\s*>\(", nm)
        if m:
            seen[(TYPE_TAGS[m.group(2)], bool(m.group(1)))] = threads[mangled]
    assert {t for t, _ in seen} == set(GRU_PROGRAMS) and len(seen) == 14
    assert set(seen.values()) == {32 * GRU_WARPS}


def test_refusals_without_a_device():
    """the softmax mode, and rnn_states with episode_length, are refused before the env is bound"""
    env = make_product_env("simple_spread_n3", num_envs=64)
    a = make_rmappo_actor(18, 5, False, True, device="cpu")
    with pytest.raises(NotImplementedError, match="categorical"):
        env.rollout_policy([a] * 3, 4)
    with pytest.raises(ValueError, match="episode_length"):
        env.rollout_policy([a] * 3, 4, action_mode="categorical", episode_length=2, rnn_states=torch.zeros(3, 64, 64))
