"""CPU checks of MAPPO's actor in the in-kernel rollout (env.rollout_policy with LayerNorm policies): mappo_actor_params
accepts exactly MAPPO's layer list and folds each LayerNorm's affine exactly; the float64 model the GPU tests judge the
kernel by agrees with an independent torch formulation; the two C entry points are declared, bound and refuse what they
can refuse without a device as the categorical ones do; and every one of the 34 kernels is compiled for the block size
the test mirror expects."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from helpers import make_product_env
from mappo_helpers import FEATURE_NORM, TANH, MappoModel, make_mappo_actors, mappo_block_cap, module_logits
from mlp_programs import PROGRAMS

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


BAD_ARG, NO_DEVICE = -1, -5


def _call(name, handle, steps=4, weights=True, hidden=64):
    from multiagent_particle_envs_b200 import _lib
    lib = _lib.load()
    argtypes = _lib._SIGNATURES[name][1]
    per_agent = _lib.ptr_array([256] * _lib.MPE_MAX_AGENTS)
    args = [256 if t is _lib._P else per_agent if t is _lib._PP else 1 if t.__name__ == "c_int" else 0 for t in argtypes]
    args[0], args[-1] = handle, None
    args[5:11] = [per_agent if weights else None] * 6
    args[11], args[12] = hidden, steps
    return getattr(lib, name)(*args)


def test_return_codes_without_a_device_are_the_categorical_ones():
    shapes = make_product_env("simple_spread_n3", num_envs=64).world.native_shapes()   # device-less handle
    handle = shapes.handle          # `shapes` owns it: the handle stays live while the test holds `shapes`
    for name, base in ENTRY_POINTS.items():
        episodes = name.endswith("_episodes")
        for hidden in (64, 32):
            probes = [dict(handle=None), dict(handle=handle, steps=-1), dict(handle=handle, weights=False),
                      dict(handle=handle)]
            want = [BAD_ARG, NO_DEVICE if episodes else BAD_ARG, NO_DEVICE if episodes else BAD_ARG, NO_DEVICE]
            for kw, w in zip(probes, want):
                assert _call(name, hidden=hidden, **kw) == _call(base, hidden=hidden, **kw) == w, (name, hidden, kw)


# ---- launch bounds ----------------------------------------------------------------------------------------------------
TYPE_TAGS = {
    "Simple<1, 1>": "simple", "Spread<2>": "simple_spread_n2", "Spread<3>": "simple_spread_n3",
    "Spread<4>": "simple_spread_n4", "Spread<5>": "simple_spread_n5", "Spread<6>": "simple_spread_n6",
    "Tag<3, 1, 2>": "simple_tag", "Tag<1, 1, 2>": "simple_tag_1v1", "Tag<2, 1, 2>": "simple_tag_2v1",
    "Tag<4, 2, 2>": "simple_tag_4v2", "Tag<6, 2, 3>": "simple_tag_6v2", "Adversary<1, 2, 2>": "simple_adversary",
    "Adversary<1, 3, 3>": "simple_adversary_n4", "Push<1, 1, 2>": "simple_push",
    "SpeakerListener": "simple_speaker_listener", "Reference": "simple_reference", "Crypto": "simple_crypto",
}


def _max_threads(lib_path):
    """mangled kernel name -> EIATTR_MAX_THREADS of `cuobjdump -elf` (the toolkit of the nvcc that builds the library)"""
    nvcc = shutil.which(os.environ.get("NVCC", "nvcc"))
    tool = None
    for d in ([os.path.dirname(os.path.realpath(nvcc))] if nvcc else []) + \
            [os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin")]:
        if os.access(os.path.join(d, "cuobjdump"), os.X_OK):
            tool = os.path.join(d, "cuobjdump")
            break
    if tool is None:
        pytest.skip("no CUDA toolkit (cuobjdump) to read the library with")
    text = subprocess.run([tool, "-elf", lib_path], capture_output=True, text=True, check=True).stdout
    out, cur, attr = {}, None, False
    for ln in text.splitlines():
        if ln.startswith("."):
            cur = ln[len(".nv.info."):] if ln.startswith(".nv.info.") else None
            attr = False
        elif cur and "Attribute:" in ln:
            attr = ln.split()[-1] == "EIATTR_MAX_THREADS"
        elif cur and attr and ln.strip().startswith("Value:"):
            out[cur] = int(ln.split()[1], 16)
            attr = False
    return out


def test_launch_bounds_are_the_mirrored_caps():
    from multiagent_particle_envs_b200 import _lib
    threads = _max_threads(_lib.LIB_PATH)
    names = list(threads)
    demangled = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True,
                               check=True).stdout.split("\n")
    seen = {}
    for mangled, nm in zip(names, demangled):
        m = re.match(r"void mpe::mpe_policy_mappo(_episode)?_kernel<mpe::(.+?)\s*>\(", nm)
        if m:
            seen[(TYPE_TAGS[m.group(2)], m.group(1) is not None)] = threads[mangled]
    assert len(seen) == 34 and {k[0] for k in seen} == set(PROGRAMS)
    assert seen == {(tag, e): 32 * mappo_block_cap(tag, e) for tag, e in seen}
