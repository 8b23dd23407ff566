"""CPU checks of MAPPO's actor in the in-kernel rollout (env.rollout_policy with LayerNorm policies): mappo_actor_params
accepts exactly MAPPO's layer list and folds each LayerNorm's affine exactly; the float64 model the GPU tests judge the
kernel by agrees with an independent torch formulation; the flip accounting the GPU tests use explains what a TF32
rounding flip or the Gumbel gap explains and nothing else; and the two C entry points are declared and bound.  Their
return codes without a device and the launch bounds of their 34 kernels are checked with the other forms' in
test_cpu_mlp_block_table.py."""
import ctypes
import os
import re

import numpy as np
import pytest

from helpers import make_product_env
from mappo_helpers import (FEATURE_NORM, TANH, MappoModel, explain_mappo_mismatches, make_mappo_actors, module_logits,
                           next_layer)
from mlp_categorical_helpers import GUMBEL_GAP, categorical_pick, log_softmax_at, split_pick_noise
from mlp_helpers import flipped, tf32_rna

torch = pytest.importorskip("torch")
nn = torch.nn
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBS, ACT = [18, 18, 18], [5, 5, 5]          # simple_spread N=3


def _params(**kw):
    from multiagent_particle_envs_b200.environment import mappo_actor_params
    return mappo_actor_params(kw.pop("pols"), kw.pop("obs", OBS), kw.pop("act", ACT))


def _seq(od=18, ad=5, H=64, act=nn.ReLU, act2=None, fn=False, order="normal", affine=True, bias=True, eps=1e-5):
    act2 = act2 or act
    ln = lambda d: nn.LayerNorm(d, eps=eps, elementwise_affine=affine)   # noqa: E731
    if order == "ln_first":        # LayerNorm before the activation
        body = [nn.Linear(od, H, bias=bias), ln(H), act(), nn.Linear(H, H), ln(H), act2(), nn.Linear(H, ad)]
    elif order == "missing":       # the second hidden LayerNorm left out
        body = [nn.Linear(od, H, bias=bias), act(), ln(H), nn.Linear(H, H), act2(), nn.Linear(H, ad)]
    else:
        body = [nn.Linear(od, H, bias=bias), act(), ln(H), nn.Linear(H, H), act2(), ln(H), nn.Linear(H, ad)]
    return nn.Sequential(*(([ln(od)] if fn else []) + body))


@pytest.mark.parametrize("tanh", [False, True])
@pytest.mark.parametrize("fn", [False, True])
def test_accepts_the_four_shapes(tanh, fn):
    pols = make_mappo_actors(OBS, ACT, tanh, fn, device="cpu")
    params, got_tanh, got_fn, eps = _params(pols=pols)
    assert (got_tanh, got_fn, eps) == (tanh, fn, 1e-5)
    assert [tuple(tuple(t.shape) for t in p) for p in params] == [((64, 18), (64,), (64, 64), (64,), (5, 64), (5,))] * 3
    assert all(t.dtype == torch.float64 for p in params for t in p)


def test_a_shared_module_is_accepted():
    m = make_mappo_actors(OBS[:1], ACT[:1], False, True, device="cpu")[0]
    params, _, _, _ = _params(pols=[m, m, m])
    for p in params[1:]:
        for x, y in zip(p, params[0]):
            assert torch.equal(x, y)


@pytest.mark.parametrize("pols,match", [
    ([_seq(order="ln_first")] * 3, "must be"),
    ([_seq(order="missing")] * 3, "must be"),
    ([_seq(affine=False)] * 3, "elementwise_affine"),
    ([_seq(act=nn.ReLU, act2=nn.Tanh)] * 3, "must be"),
    ([_seq(act=nn.ReLU), _seq(act=nn.Tanh), _seq(act=nn.ReLU)], "same activation"),
    ([_seq(eps=1e-5), _seq(eps=1e-5), _seq(eps=1e-6)], "same eps"),
    ([_seq(fn=True), _seq(fn=False), _seq(fn=True)], "every policy or for none"),
    ([_seq(H=32)] * 3, "hidden width 64"),
    ([_seq(H=128)] * 3, "hidden width 64"),
    ([_seq(bias=False)] * 3, "bias"),
    ([_seq(od=17)] * 3, "expected"),
    ([_seq(ad=6)] * 3, "expected"),
    ([_seq(act=nn.GELU)] * 3, "must be"),
    ([_seq()] * 2, "expected 3 policies"),
    ([_seq()] * 4, "expected 3 policies"),
])
def test_refuses_other_networks(pols, match):
    with pytest.raises(ValueError, match=match):
        _params(pols=pols)


def test_refuses_a_bare_module_list():
    m = _seq()
    with pytest.raises(ValueError, match="must be"):
        _params(pols=[nn.ModuleList(list(m))] * 3)


def _folded_forward(params, obs, tanh, fn, eps):
    """the folded network with parameter-free LayerNorms, float64"""
    def ln(x):
        mu = x.mean(-1, keepdims=True)
        return (x - mu) / np.sqrt(((x - mu) ** 2).mean(-1, keepdims=True) + eps)
    act = np.tanh if tanh else (lambda v: np.maximum(v, 0.0))
    W1, b1, W2, b2, W3, b3 = [t.numpy() for t in params]
    x = ln(obs) if fn else obs
    x = ln(act(x @ W1.T + b1))
    x = ln(act(x @ W2.T + b2))
    return x @ W3.T + b3


@pytest.mark.parametrize("tanh", [False, True])
@pytest.mark.parametrize("fn", [False, True])
def test_the_fold_is_exact(tanh, fn):
    pols = make_mappo_actors(OBS, ACT, tanh, fn, device="cpu", eps=1e-3)
    params, _, _, eps = _params(pols=pols)
    obs = np.random.RandomState(0).randn(512, 18) * 2.0
    for m, p in zip(pols, params):
        np.testing.assert_allclose(_folded_forward(p, obs, tanh, fn, eps), module_logits(m, obs), rtol=0, atol=1e-12)


def _tf32_torch(x):
    """fp32 -> TF32, ties away from zero, in torch integer arithmetic (independent of mlp_helpers.tf32_rna)"""
    b = x.to(torch.float32).view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    exp_all_ones = (b & 0x7F800000) == 0x7F800000
    r = torch.where(exp_all_ones, b, (b + 0x1000) & 0xFFFFE000)
    r = torch.where(r >= 2 ** 31, r - 2 ** 32, r)
    return r.to(torch.int32).view(torch.float32).to(torch.float64)


@pytest.mark.parametrize("tanh", [False, True])
@pytest.mark.parametrize("fn", [False, True])
def test_model_is_the_torch_float64_recipe(tanh, fn):
    """MappoModel (normalise in float64, round the operand to TF32, GEMM in float64 with TF32 weights and fp32 biases)
    against the same recipe written with torch.nn.functional"""
    F = torch.nn.functional
    pols = make_mappo_actors(OBS, ACT, tanh, fn, device="cpu")
    params, _, _, eps = _params(pols=pols)
    net = ((FEATURE_NORM if fn else 0) | (TANH if tanh else 0), eps)
    obs = np.random.RandomState(1).randn(1024, 18).astype(np.float32) * 1.5
    act = torch.tanh if tanh else torch.relu
    for p in params:
        p32 = [t.to(torch.float32) for t in p]
        model = MappoModel([t.numpy() for t in p32], net)
        W = [_tf32_torch(p32[j]) for j in (0, 2, 4)]
        b = [p32[j].to(torch.float64) for j in (1, 3, 5)]
        x = torch.as_tensor(obs, dtype=torch.float64)
        if fn:
            x = F.layer_norm(x, (18,), eps=eps)
        x = _tf32_torch(x)
        for j in range(2):
            x = _tf32_torch(F.layer_norm(act(F.linear(x, W[j], b[j])), (64,), eps=eps))
        want = F.linear(x, W[2], b[2]).numpy()
        np.testing.assert_allclose(model(obs), want, rtol=0, atol=1e-12)


# ---- explain_mappo_mismatches on a synthetic actor (no GPU) -----------------------------------------------------------
def _model_and_obs():
    """agent 0's folded actor with the input LayerNorm, and 32 observations"""
    params, _, _, eps = _params(pols=make_mappo_actors(OBS, ACT, False, True, device="cpu"))
    model = MappoModel([t.to(torch.float32).numpy() for t in params[0]], (FEATURE_NORM, eps))
    return model, np.random.RandomState(5).uniform(-2.0, 2.0, (32, 18)).astype(np.float32)


def test_accounting_explains_a_pick_moved_by_a_tf32_flip_and_one_within_the_gumbel_gap():
    model, obs = _model_and_obs()
    segs = [5]
    z = model(obs)
    # the "kernel" rounds one ambiguous group of row 11's x2 the other way: the one that moves a pair of logits furthest
    # apart.  x1 and x2 are evaluated one row at a time, as the accounting does
    x0 = tf32_rna(model.input(obs)[0].astype(np.float32)).astype(np.float64)
    r1, _, _ = next_layer(model, 0)(x0[11])
    r2, alt2, groups = next_layer(model, 1)(r1)
    zk = max((model.logits(flipped(r2, alt2, [g])) for g in groups), key=lambda v: np.ptp(v - z[11]))
    noise = np.zeros_like(z)
    noise[11], pick11, half = split_pick_noise(z[11], zk)
    assert half > 1e-4                      # the pick moves, and by more than the Gumbel gap
    a, b = np.argsort(z[3])[::-1][:2]       # row 3: the runner-up within the Gumbel gap of the pick
    noise[3, b] = z[3, a] - z[3, b] - GUMBEL_GAP / 2
    k = categorical_pick(z + noise, segs)
    logp = log_softmax_at(z, k, segs)
    assert explain_mappo_mismatches(k, logp, obs, model, segs, noise=noise) == (0, 0)
    assert k[11, 0] != pick11 and k[3, 0] == a
    k[11, 0], k[3, 0] = pick11, b
    logp = log_softmax_at(z, k, segs)
    logp[11] = log_softmax_at(zk[None], k[11:12], segs)[0]
    assert explain_mappo_mismatches(k, logp, obs, model, segs, noise=noise) == (1, 1)


def test_accounting_rejects_a_wrong_pick_and_a_wrong_log_probability():
    model, obs = _model_and_obs()
    segs = [5]
    z = model(obs)
    k = categorical_pick(z, segs)
    logp = log_softmax_at(z, k, segs)
    assert explain_mappo_mismatches(k, logp, obs, model, segs) == (0, 0)
    bad = k.copy()
    bad[7, 0] = np.argmin(z[7])             # with the model's log-probability of that pick
    with pytest.raises(AssertionError, match="neither TF32 rounding flips of the normalised operands nor within"):
        explain_mappo_mismatches(bad, log_softmax_at(z, bad, segs), obs, model, segs)
    wrong = logp.copy()
    wrong[7] += 1e-2
    with pytest.raises(AssertionError, match=r"\(7, "):
        explain_mappo_mismatches(k, wrong, obs, model, segs)


def test_refusals_without_a_device():
    """the softmax mode and a hidden width other than 64 are refused before the env is bound"""
    env = make_product_env("simple_spread_n3", num_envs=64)
    obs_dims = env.world.native_shapes().obs_dims                 # device-less handle
    pols = make_mappo_actors(obs_dims, [5] * 3, False, True, device="cpu")
    with pytest.raises(NotImplementedError, match="categorical"):
        env.rollout_policy(pols, 4)
    with pytest.raises(NotImplementedError, match="categorical"):
        env.rollout_policy(pols, 4, action_mode="softmax", explore_seed=1)
    h32 = make_mappo_actors(obs_dims, [5] * 3, True, False, device="cpu", hidden=32)
    with pytest.raises(NotImplementedError, match="hidden width 64"):
        env.rollout_policy(h32, 4, action_mode="categorical")
    with pytest.raises(ValueError, match="record_log_probs"):
        env.rollout_policy(pols, 4, record_log_probs=True)


# ---- the C entry points --------------------------------------------------------------------------------------------
ENTRY_POINTS = {"mpe_rollout_policy_mappo": "mpe_rollout_policy_mlp_categorical",
                "mpe_rollout_policy_mappo_episodes": "mpe_rollout_policy_mlp_categorical_episodes"}


def test_entry_points_are_declared_exported_and_bound():
    from multiagent_particle_envs_b200 import _lib
    header = open(os.path.join(ROOT, "include", "mpe_b200.h")).read()
    declared = set(re.findall(r"MPE_API[^;(]*?\b(mpe_[a-z_]+)\s*\(", header))
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name, base in ENTRY_POINTS.items():
        assert name in declared and name in _lib.EXPORTED_SYMBOLS and hasattr(lib, name), name
        # the categorical form's parameters with (net_flags, ln_eps) before (done, flags, stream)
        got, want = _lib._SIGNATURES[name][1], list(_lib._SIGNATURES[base][1])
        assert got == want[:-3] + [ctypes.c_uint32, ctypes.c_float] + want[-3:], name
    assert _lib.MPE_ABI_VERSION == 1
