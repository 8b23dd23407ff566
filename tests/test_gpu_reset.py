"""The reset draw of every compiled program, bit for bit against a NumPy model of draw_initial_state
(csrc/mpe_kernels.cu): agents ~ U(-1, 1)^2 at rest, landmarks ~ U(-r, r)^2, utterances 0, goal g = word g of Philox
block 0x80000000 mod the landmark count.  One Philox4x32-10 block holds two entities' (x, y), entities in the order
agents then landmarks; key = seed (lo, hi), counter = (global world index lo, hi, low 32 bits of epoch, entity pair).
The episode forms of the rollout kernels redraw through the same function and equal a loop of env.reset() calls bit for
bit, so this also pins the in-kernel redraw."""
import numpy as np
import pytest

from helpers import CONFIGS, PROGRAM_TAGS, VARIANTS, make_product_env, random_actions, split_cols
from mlp_helpers import philox4x32_10

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

GOAL_BLOCK = 0x80000000
# what reset_world draws, per scenario, read from the reference (not from this library): landmark half-width, and the
# goal words (each one a landmark index; crypto's second word is the key, np.random.choice(world.landmarks).color, whose
# one-hot color is that landmark's index -- make_golden.goals_of).  Agents are U(-1, 1) in every scenario
# (e.g. simple_spread.py:40, simple_tag.py:48, simple_world_comm.py:102).
RESET_TABLE = {
    "simple": (1.0, 0),                       # simple.py:38
    "simple_spread": (1.0, 0),                # simple_spread.py:44
    "simple_tag": (0.9, 0),                   # simple_tag.py:53
    "simple_world_comm": (0.9, 0),            # simple_world_comm.py:106, :109, :112 (landmarks, food, forests)
    "simple_adversary": (1.0, 1),             # simple_adversary.py:44 (goal), :54
    "simple_push": (1.0, 1),                  # simple_push.py:40 (goal), :55
    "simple_speaker_listener": (1.0, 1),      # simple_speaker_listener.py:40 (goal_b), :56
    "simple_reference": (1.0, 2),             # simple_reference.py:33, :35 (goal_b of both agents), :52
    "simple_crypto": (1.0, 2),                # simple_crypto.py:61 (goal), :63 (key), :74
}


def uniform_from_bits(bits, lo, hi):
    """lo + (hi - lo) * ((bits >> 8) * 2^-24) in fp32 as reset_kernel computes it: nvcc contracts it into one
    FFMA(hi - lo, u, lo) (cuobjdump -sass of reset_kernel), and hi - lo = 2 r is exact.  (hi - lo) * u needs at most 48
    bits and the sum with lo stays on the same 2^-47 grid below 2, so the float64 evaluation is exact and one rounding
    to float32 is the FFMA's."""
    u = (np.asarray(bits, np.uint32) >> 8).astype(np.float64) * 2.0 ** -24
    lo32, width32 = np.float32(lo), np.float32(hi) - np.float32(lo)
    return (np.float64(lo32) + np.float64(width32) * u).astype(np.float32)


def draw_initial_state(seed, gw, epoch, A, L, G, landmark_range, goal_mod):
    """(agent positions [A, n, 2], landmark positions [L, n, 2], goals [G, n]) for the global world indices gw"""
    gw = np.asarray(gw, np.uint64)
    key = (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)

    def block(word3):
        ctr = np.stack([gw & np.uint64(0xFFFFFFFF), gw >> np.uint64(32), np.full_like(gw, epoch & 0xFFFFFFFF),
                        np.full_like(gw, word3)], -1)
        return philox4x32_10(ctr, key)

    pos = []
    for e in range(A + L):
        r = block(e >> 1)
        k = e & 1
        lim = 1.0 if e < A else landmark_range
        pos.append(np.stack([uniform_from_bits(r[:, 2 * k], -lim, lim), uniform_from_bits(r[:, 2 * k + 1], -lim, lim)],
                            -1))
    goal = (block(GOAL_BLOCK)[:, :G] % np.uint32(goal_mod)).T.astype(np.int32)
    return np.array(pos[:A]), np.array(pos[A:]), goal


def check_draw(env, tag, seed, epoch, worlds):
    """the worlds selected by `worlds` (bool [n]) hold the model's draw at (seed, world_offset + w, epoch)"""
    nw = env.world.native
    A, L, G = nw.n_agents, nw.n_landmarks, nw.n_goals
    rng_half, n_goals = RESET_TABLE[(CONFIGS[tag] if tag in CONFIGS else VARIANTS[tag])[0]]
    assert G == n_goals
    gw = nw.world_offset + np.arange(nw.n_env, dtype=np.uint64)[worlds]
    ap, lp, goal = draw_initial_state(seed, gw, epoch, A, L, G, rng_half, L)
    pv = nw.agent_pv.cpu().numpy()[:, worlds]
    assert np.array_equal(pv[:, :, 0:2].view(np.uint32), ap.view(np.uint32))
    assert np.array_equal(pv[:, :, 2:4], np.zeros_like(pv[:, :, 2:4]))
    assert np.array_equal(nw.lm_p[:L].cpu().numpy()[:, worlds].view(np.uint32), lp.view(np.uint32))
    if nw.n_speakers and nw.dim_c:
        assert not nw.comm.cpu().numpy()[:, worlds].any()
    if G:
        assert np.array_equal(nw.goal.cpu().numpy()[:, worlds], goal)


@pytest.mark.parametrize("tag", PROGRAM_TAGS)
def test_reset_draw_is_the_model(tag):
    """a seed >= 2^32; later epochs (each reset advances it; building the env draws epoch 0); world_offset 2^32 + 5 (the
    counter's high word 1); a masked reset after a step, which redraws the masked worlds and leaves every other one
    untouched bit for bit"""
    n, seed = 1000, 0x1_2345_6789
    env = make_product_env(tag, num_envs=n, seed=seed)
    nw = env.world.native
    every = np.ones(n, bool)

    def reset_and_check(mask=None):
        epoch = nw.epoch                                   # the epoch this reset draws with
        env.reset() if mask is None else env.reset(mask=torch.as_tensor(mask, device="cuda"))
        check_draw(env, tag, seed, epoch, every if mask is None else mask)
        return epoch

    first = reset_and_check()
    env.reset()
    assert reset_and_check() == first + 2
    nw.world_offset = 2 ** 32 + 5
    reset_and_check()
    nw.world_offset = 0
    # a step moves every world and sets the utterances; then a masked reset
    rng = np.random.RandomState(2)
    desc = env.world.descriptor()
    act = random_actions(nw.act_dims, n, rng, movable=[bool(desc.agent_movable[i]) for i in range(desc.n_agents)])
    env.step([torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32, device="cuda")
              for a in split_cols(act.astype(np.float32), nw.act_dims)])
    before = [t.clone() for t in (nw.agent_pv, nw.lm_p, nw.comm, nw.goal)]
    mask = rng.uniform(0, 1, n) < 0.4
    reset_and_check(mask)
    keep = torch.as_tensor(~mask, device="cuda")
    for b, t in zip(before, (nw.agent_pv, nw.lm_p, nw.comm, nw.goal)):
        assert torch.equal(b[:, keep], t[:, keep])
