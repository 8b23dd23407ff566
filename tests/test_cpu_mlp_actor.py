"""CPU checks of the two-hidden-layer in-kernel actor's host side: the NumPy TF32 rounding and Philox4x32-10 models the
GPU tests compare against, and the Python-side validation of malformed Linear-ReLU-Linear-ReLU-Linear policies."""
import numpy as np
import pytest

from helpers import make_product_env
import mlp_helpers
from mlp_helpers import dyadic_actor, philox4x32_10, softmax, tf32_rna, tf32_rne, tf32_tie, uniform_from_bits

torch = pytest.importorskip("torch")


def _f(bits):
    return np.array([bits], dtype=np.uint32).view(np.float32)[0]


def test_tf32_round_to_nearest_ties_away():
    one = 1.0
    cases = [
        (one, one),
        (one + 2 ** -11, one + 2 ** -10),                 # exact tie: away from zero (nearest-even would give 1.0)
        (-(one + 2 ** -11), -(one + 2 ** -10)),
        (one + 2 ** -11 - 2 ** -23, one),                  # just below the tie
        (one + 3 * 2 ** -11, one + 2 ** -9),               # tie between 1 + 2^-10 and 1 + 2^-9
        (2.0 - 2 ** -23, 2.0),                             # mantissa carry into the exponent
        (-(2.0 - 2 ** -23), -2.0),
        (0.0, 0.0),
        (1.5 + 2 ** -12, 1.5),                             # below half a unit
    ]
    for x, want in cases:
        got = tf32_rna(np.float32(x))
        assert got == np.float32(want), (x, got, want)
    assert tf32_rna(_f(0x00001000)).view(np.uint32) == 0x00002000      # subnormal tie rounds up
    assert tf32_rna(_f(0x7F7FF000)).view(np.uint32) == 0x7F800000      # largest tie overflows to +inf
    assert np.isnan(tf32_rna(np.float32(np.nan))) and tf32_rna(np.float32(np.inf)) == np.inf
    x = np.random.RandomState(0).randn(1000).astype(np.float32)
    r = tf32_rna(x)
    assert (r.view(np.uint32) & 0x1FFF == 0).all() and np.abs(r - x).max() <= np.abs(x).max() * 2 ** -11


def test_philox_known_answers():
    # Random123's known-answer vectors for Philox4x32-10
    assert philox4x32_10([0, 0, 0, 0], (0, 0)).tolist() == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    assert philox4x32_10([0xFFFFFFFF] * 4, (0xFFFFFFFF, 0xFFFFFFFF)).tolist() == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]
    assert philox4x32_10([0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344], (0xA4093822, 0x299F31D0)).tolist() == \
        [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]
    batch = philox4x32_10(np.array([[1, 2, 3, 4], [0, 0, 0, 0]], dtype=np.uint32), (0, 0))
    assert batch[1].tolist() == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]


def test_uniforms_stay_inside_the_open_interval():
    u = uniform_from_bits(np.array([0, 0xFF, 0x7FFFFF00, 0xFFFFFFFF], dtype=np.uint32))
    assert u[0] == np.float32(2.0 ** -25) and u[1] == u[0]
    assert u[2] == np.float32((0x7FFFFF + 0.5) * 2.0 ** -24)
    assert u[3] == np.float32(1 - 2.0 ** -24) and (u < 1).all() and (u > 0).all()


def _mods(obs_dims, H, layers):
    return [torch.nn.Sequential(*layers(od, H)) for od in obs_dims]


def test_malformed_two_hidden_layer_policies_are_refused():
    from multiagent_particle_envs_b200.environment import mlp_actor_params, _has_two_hidden_layers
    nn = torch.nn
    env = make_product_env("simple_spread_n3", num_envs=64)
    obs_dims = env.world.native_shapes().obs_dims               # device-less handle
    assert obs_dims == [18, 18, 18]
    good = _mods(obs_dims, 64, lambda od, H: [nn.Linear(od, H), nn.ReLU(), nn.Linear(H, H), nn.ReLU(), nn.Linear(H, 5)])
    params, H = mlp_actor_params(good, obs_dims)
    assert H == 64 and len(params) == 3 and [tuple(t.shape) for t in params[0]] == [(64, 18), (64,), (64, 64), (64,), (5, 64), (5,)]
    assert all(_has_two_hidden_layers(m) for m in good)
    tuples = [tuple(p) for p in params]
    assert mlp_actor_params(tuples, obs_dims)[1] == 64
    bad = {
        "order": lambda od, H: [nn.Linear(od, H), nn.Linear(H, H), nn.ReLU(), nn.ReLU(), nn.Linear(H, 5)],
        "tanh": lambda od, H: [nn.Linear(od, H), nn.Tanh(), nn.Linear(H, H), nn.ReLU(), nn.Linear(H, 5)],
        "leaky": lambda od, H: [nn.Linear(od, H), nn.ReLU(), nn.Linear(H, H), nn.LeakyReLU(), nn.Linear(H, 5)],
        "extra": lambda od, H: [nn.Linear(od, H), nn.ReLU(), nn.Linear(H, H), nn.ReLU(), nn.Linear(H, 5), nn.Softmax(-1)],
        "widths": lambda od, H: [nn.Linear(od, H), nn.ReLU(), nn.Linear(H, 32), nn.ReLU(), nn.Linear(32, 5)],
        "obs_dim": lambda od, H: [nn.Linear(od + 1, H), nn.ReLU(), nn.Linear(H, H), nn.ReLU(), nn.Linear(H, 5)],
        "outputs": lambda od, H: [nn.Linear(od, H), nn.ReLU(), nn.Linear(H, H), nn.ReLU(), nn.Linear(H, 4)],
        "no_bias": lambda od, H: [nn.Linear(od, H), nn.ReLU(), nn.Linear(H, H, bias=False), nn.ReLU(), nn.Linear(H, 5)],
    }
    for name, layers in bad.items():
        mods = _mods(obs_dims, 64, layers)
        assert _has_two_hidden_layers(mods[0]), name
        with pytest.raises(ValueError):
            mlp_actor_params(mods, obs_dims)
    with pytest.raises(ValueError, match="W1 \\[64, 18\\]"):           # the message names the expected shapes
        mlp_actor_params(_mods(obs_dims, 64, bad["widths"]), obs_dims)
    mixed = [good[0], good[1], _mods(obs_dims, 32, lambda od, H: [nn.Linear(od, H), nn.ReLU(), nn.Linear(H, H), nn.ReLU(),
                                                                  nn.Linear(H, 5)])[0]]
    with pytest.raises(ValueError):                                  # one hidden width for all agents
        mlp_actor_params(mixed, obs_dims)
    with pytest.raises(ValueError):                                  # a module that is not a Sequential
        class Net(nn.Module):
            def __init__(self):
                super().__init__()
                self.a, self.b, self.c = nn.Linear(18, 64), nn.Linear(64, 64), nn.Linear(64, 5)
        mlp_actor_params([Net(), good[1], good[2]], obs_dims)
    with pytest.raises(ValueError):
        mlp_actor_params(tuples[:2], obs_dims)                       # one policy per agent
    with pytest.raises(ValueError):
        mlp_actor_params([tuples[0][:5] + (torch.zeros(4),), tuples[1], tuples[2]], obs_dims)
    # one-hidden-layer policies keep their own path
    one = nn.Sequential(nn.Linear(18, 64), nn.ReLU(), nn.Linear(64, 5))
    assert not _has_two_hidden_layers(one) and not _has_two_hidden_layers(tuples[0][:4])


# ---- explain_tf32_mismatches on synthetic actors (no GPU) ----------------------------------------------------------
def _actions(obs, params, rnd=tf32_rna, h1_override=None):
    """the actor with every operand rounded by `rnd` and exact accumulation; h1_override (row, unit, value) replaces
    one rounded h1 entry"""
    f64 = np.float64
    W1, b1, W2, b2, W3, b3 = params
    h1 = rnd(np.maximum(rnd(obs).astype(f64) @ rnd(W1).astype(f64).T + b1, 0).astype(np.float32)).astype(f64)
    if h1_override is not None:
        h1[h1_override[0], h1_override[1]] = h1_override[2]
    h2 = rnd(np.maximum(h1 @ rnd(W2).astype(f64).T + b2, 0).astype(np.float32)).astype(f64)
    return softmax(h2 @ rnd(W3).astype(f64).T + b3)


def test_accounting_accepts_a_unit_on_a_tf32_midpoint_rounded_the_other_way():
    rng = np.random.RandomState(1)
    obs, (W1, b1, W2, b2, W3, b3) = dyadic_actor(rng)
    # unit 0 of row 5: pre-activation 1 + 2^-11 exactly (a TF32 tie); the model rounds it up to 1 + 2^-10, the "kernel"
    # lands a hair below the tie and rounds it down to 1
    W1 = W1.copy()
    W1[0] = 0.0
    b1 = b1.copy()
    b1[0] = np.float32(1 + 2 ** -11)
    W2 = W2.copy()
    W2[:, 0] = 1.0                          # make the flip visible in the actions
    params = (W1, b1, W2, b2, W3, b3)
    want = _actions(obs, params)
    got = _actions(obs, params, h1_override=(5, 0, 1.0))
    assert np.abs(got - want)[5].max() > 1e-4 and np.abs(got - want)[np.arange(32) != 5].max() == 0
    assert mlp_helpers.explain_tf32_mismatches(got, obs, params) == 1
    assert mlp_helpers.explain_tf32_mismatches(want, obs, params) == 0


def test_accounting_rejects_a_perturbation_without_an_ambiguous_unit():
    obs, params = dyadic_actor(np.random.RandomState(2))
    got = _actions(obs, params)
    assert mlp_helpers.explain_tf32_mismatches(got, obs, params) == 0
    bad = got.copy()
    bad[7, 2] += 3e-4
    with pytest.raises(AssertionError, match="not TF32 rounding flips"):
        mlp_helpers.explain_tf32_mismatches(bad, obs, params)
    # a wrong logit, renormalised by the softmax as a lane bug would be
    z = mlp_helpers.actor_logits(obs, *params)
    z[7, z[7].argmax()] += 2e-3
    bad = got.copy()
    bad[7] = softmax(z[7])
    assert np.abs(bad - got).max() > 1e-4
    with pytest.raises(AssertionError, match="not TF32 rounding flips"):
        mlp_helpers.explain_tf32_mismatches(bad, obs, params)


def test_accounting_rejects_a_perturbation_in_the_last_row_of_a_tile():
    """generic weights (ambiguous units everywhere): a change no rounding flip can make -- one entry of the last row of
    a 32-row tile, so the row no longer sums to one -- is still caught"""
    rng = np.random.RandomState(3)
    od, H = 18, 64
    r = lambda *s: rng.randn(*s).astype(np.float32)                                     # noqa: E731
    params = (r(H, od) * 1.5 / od ** 0.5, r(H) * 0.3, r(H, H) * 1.5 / H ** 0.5, r(H) * 0.3, r(5, H) * 1.5 / H ** 0.5,
              r(5) * 0.2)
    obs = rng.uniform(-1.5, 1.5, (64, od)).astype(np.float32)
    got = _actions(obs, params)
    mlp_helpers.explain_tf32_mismatches(got, obs, params)
    bad = got.copy()
    bad[31, 4] += 1e-4
    with pytest.raises(AssertionError, match=r"\(31, "):
        mlp_helpers.explain_tf32_mismatches(bad, obs, params)
    z = mlp_helpers.actor_logits(obs, *params)                  # a wrong logit of that row, renormalised
    z[31, 4] += 4e-3
    bad = got.copy()
    bad[31] = softmax(z[31])
    assert np.abs(bad - got).max() > 3e-4
    with pytest.raises(AssertionError, match=r"\(31, "):
        mlp_helpers.explain_tf32_mismatches(bad, obs, params)


def test_accounting_rejects_round_to_nearest_even():
    """weights and observations that are exact TF32 ties: an actor that rounds them to nearest-even is not the kernel"""
    rng = np.random.RandomState(4)
    obs, (W1, b1, W2, b2, W3, b3) = dyadic_actor(rng)
    params = (tf32_tie(W1 + 0.3), b1, tf32_tie(W2 + 0.1), b2, tf32_tie(W3), b3)
    obs = tf32_tie(obs + 0.7)
    assert (tf32_rna(params[0]) != tf32_rne(params[0])).mean() > 0.3
    want = _actions(obs, params)
    assert mlp_helpers.explain_tf32_mismatches(want, obs, params) == 0
    rne = _actions(obs, params, rnd=tf32_rne)
    assert np.abs(rne - want).max() > 1e-4
    with pytest.raises(AssertionError, match="not TF32 rounding flips"):
        mlp_helpers.explain_tf32_mismatches(rne, obs, params)


def test_regime_sizes_match_the_launch_rules():
    """the batch sizes the GPU tests use for each launch-shape regime, for an H100 SXM (132 SMs) and PCIe (114 SMs)"""
    from helpers import launch_shape, regime_size, step_uses_dense
    for sms in (132, 114):
        for kernel, wpbs in (("step", (1, 2, 4)), ("rollout", (1, 2, 4)), ("policy", (1, 2, 4)), ("mlp", (1, 5, 12, 16))):
            for wpb in wpbs:
                n = regime_size(kernel, sms, wpb, base=2048 if wpb == 1 else None)
                got = launch_shape(kernel, n, sms)
                assert got[0] == wpb and got[2] == (wpb > 1) and got[3] == 17, (sms, kernel, wpb, n, got)
        n = regime_size("mlp", sms, 12, cap=12, base=65536)
        assert n > 65536 and launch_shape("mlp", n, sms, cap=12)[0] == 12 and launch_shape("mlp", n, sms)[0] == 16
        assert step_uses_dense("simple_tag", regime_size("step", sms, 2), sms)
        assert not step_uses_dense("simple_spread_n6", regime_size("step", sms, 2), sms)
    # the thresholds themselves, at 132 SMs
    assert launch_shape("step", 16 * 132 * 32 + 31, 132)[0] == 1 and launch_shape("step", (16 * 132 + 1) * 32, 132)[0] == 2
    assert launch_shape("rollout", 4 * 132 * 32, 132)[0] == 1 and launch_shape("rollout", 4 * 132 * 32 + 1, 132)[0] == 2
    assert launch_shape("policy", 64 * 132 * 32, 132)[0] == 2 and launch_shape("policy", 64 * 132 * 32 + 1, 132)[0] == 4
    assert launch_shape("mlp", 65536, 132) == (16, 128, False, 32)
    assert launch_shape("mlp", 65536, 132, cap=12) == (12, 171, True, 32)
    assert launch_shape("mlp", 65536, 114) == (16, 128, False, 32)
