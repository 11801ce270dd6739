"""The per-engine render launch keys ("obs_grid", "obs_chunk", "obs_tile") and the "obs_launch" report, on the host
emulation (tests/emu/): the keys are stored per engine and refused when invalid, and a backend that does not report
its render launches refuses "obs_launch" instead of failing."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import parity_common as pc

KEYS = (b"obs_grid", b"obs_chunk", b"obs_tile")


@pytest.fixture(scope="module")
def emu():
    src_dir = os.path.join(pc.REPO, "magent_b200", "csrc")
    newest = max(os.path.getmtime(os.path.join(src_dir, f)) for f in os.listdir(src_dir))
    newest = max(newest, os.path.getmtime(os.path.join(pc.REPO, "tests", "emu", "backend_emu.cc")))
    if not os.path.exists(pc.EMU_LIB) or os.path.getmtime(pc.EMU_LIB) < newest:
        subprocess.run([os.path.join(pc.REPO, "tests", "emu", "build.sh")], check=True, capture_output=True)
    return pc.EMU_LIB


def config(env, key, value):
    return env._lib.env_config_game(env.game, key, ctypes.byref(ctypes.c_int(value)))


def test_keys_are_stored_per_engine_and_change_between_calls(emu):
    a = pc.make_battle(emu, 24, 30, 1, _obs_launch=(3, 8, 2))
    b = pc.make_battle(emu, 24, 30, 1)
    assert a._get_obs_override() == (3, 8, 2)
    assert b._get_obs_override() == (0, 0, 0)
    h = a.get_handles()[0]
    first = a.get_observation(h)[0].copy()
    for key, value, want in ((b"obs_grid", 1, (1, 8, 2)), (b"obs_chunk", 0, (1, 0, 2)), (b"obs_tile", 1, (1, 0, 1))):
        assert config(a, key, value) == 0
        assert a._get_obs_override() == want
    a._set_obs_launch(0, 0, 0)
    assert a._get_obs_override() == (0, 0, 0)
    assert b._get_obs_override() == (0, 0, 0)
    np.testing.assert_array_equal(a.get_observation(h)[0].view(np.uint32), first.view(np.uint32))


@pytest.mark.parametrize("key,value", [(b"obs_grid", -1), (b"obs_chunk", -5), (b"obs_tile", -1), (b"obs_tile", 3),
                                       (b"obs_grid", -2 ** 31)])
def test_invalid_values_are_refused_and_change_nothing(emu, key, value):
    env = pc.make_battle(emu, 24, 30, 1, _obs_launch=(2, 3, 1))
    assert config(env, key, value) == -1
    why = env._lib.magent_b200_last_error().decode()
    assert key.decode() in why and str(value) in why, why
    assert env._get_obs_override() == (2, 3, 1)


def test_wrapper_refuses_as_a_whole(emu):
    env = pc.make_battle(emu, 24, 30, 1, _obs_launch=(2, 3, 1))
    with pytest.raises(ValueError, match="obs_tile"):
        env._set_obs_launch(5, 5, 3)
    assert env._get_obs_override() == (2, 3, 1)
    with pytest.raises(ValueError, match="obs_chunk"):
        pc.make_battle(emu, 24, 30, 1, _obs_launch=(1, -1, 0))


def test_obs_launch_is_refused_without_the_backend_report(emu):
    env = pc.make_battle(emu, 24, 30, 1, _obs_launch=(1, 1, 1))
    env.get_observation(env.get_handles()[0])
    buf = np.full((8,), 7, np.int32)
    assert env._lib.env_get_info(env.game, -1, b"obs_launch", buf.ctypes.data) == -1
    assert "report" in env._lib.magent_b200_last_error().decode()
    assert (buf == 7).all()
    with pytest.raises(RuntimeError, match="obs_launch refused"):
        env._get_obs_launch()


def test_reference_library_has_no_launch_keys():
    lib = pc.REF_LIB if os.path.exists(pc.REF_LIB) else pc.PORT_LIB
    if not os.path.exists(lib):
        pytest.skip("no oracle library available (oracle/_ref or oracle/_build)")
    with pytest.raises(ValueError, match="_obs_launch"):
        pc.make_battle(lib, 24, 30, 1, _obs_launch=(1, 1, 1))
