"""CPU checks of the two-hidden-layer in-kernel actor's host side: the NumPy TF32 rounding and Philox4x32-10 models the
GPU tests compare against, and the Python-side validation of malformed Linear-ReLU-Linear-ReLU-Linear policies."""
import numpy as np
import pytest

from helpers import make_product_env
from mlp_helpers import philox4x32_10, tf32_rna, uniform_from_bits

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
