"""The observation render picks its tile width per launch: 8-agent f32 tiles where they keep as many warps per SM
as 4-agent tiles, 4-agent tiles otherwise.  A record too large for an 8-agent tile in shared memory must still
render, bit-exact against the oracle."""
import os

import pytest

import parity_common as pc

pytestmark = pytest.mark.gpu

SMEM_PER_BLOCK = 227 * 1024


def checker_lib():
    for p in (pc.REF_LIB, pc.PORT_LIB):
        if os.path.exists(p):
            return p
    pytest.skip("no oracle library available (oracle/_ref or oracle/_build)")


def wide_view_config(size, radius):
    """battle with a CircleRange(radius) view: 2 groups with minimap, 7 channels"""
    import magent_b200 as magent
    gw = magent.gridworld
    cfg = gw.Config()
    cfg.set({"map_width": size, "map_height": size, "minimap_mode": True, "embedding_size": 10})
    small = cfg.register_agent_type("small", dict(
        width=1, length=1, hp=10, speed=2, damage=2, step_recover=0.1, step_reward=-0.005, kill_reward=5,
        dead_penalty=-0.1, attack_penalty=-0.1, view_range=gw.CircleRange(radius), attack_range=gw.CircleRange(1.5)))
    g0, g1 = cfg.add_group(small), cfg.add_group(small)
    a, b = gw.AgentSymbol(g0, index='any'), gw.AgentSymbol(g1, index='any')
    cfg.add_reward_rule(gw.Event(a, 'attack', b), receiver=a, value=0.2)
    cfg.add_reward_rule(gw.Event(b, 'attack', a), receiver=b, value=0.2)
    return cfg


def make_wide_view(lib, radius, map_size=48, seed=5):
    import magent_b200 as magent
    env = magent.GridWorld(wide_view_config(map_size, radius), _lib=lib)
    env.set_seed(seed)
    env.reset()
    h = env.get_handles()
    env.add_agents(h[0], method="random", n=90)
    env.add_agents(h[1], method="random", n=90)
    return env


def test_record_too_large_for_the_wide_tile_renders():
    """CircleRange(16): 33 x 33 x 7 = 7623 floats per record; a 4-agent tile fits a CTA's shared memory, an
    8-agent tile does not"""
    radius = 16
    env = make_wide_view(pc.CUDA_LIB, radius)
    h, w, c = env.get_view_space(env.get_handles()[0])
    rec_bytes = h * w * c * 4
    assert 4 * rec_bytes < SMEM_PER_BLOCK < 8 * rec_bytes
    want = pc.run_trace(make_wide_view(checker_lib(), radius), 12, 5, keep_obs=True)
    got = pc.run_trace(env, 12, 5, keep_obs=True)
    pc.compare_traces(want, got)
