"""Loader for the C-ABI engine library.

Mirrors the role of the reference loader (reference: python/magent/c_lib.py:10-42) but
 * the library is resolved in-tree (``magent_b200/lib/libmagent.so``) or from the
   ``MAGENT_B200_LIB`` environment variable / an explicit path, so the same host code can drive
   the B200 engine *or* any other library exporting the ``src/runtime_api.h`` ABI (the parity
   tests drive the compiled reference through this very wrapper);
 * every entry point gets explicit ``argtypes``/``restype`` (the reference relies on ctypes
   defaults) — the table below is the single Python-side statement of the ABI in
   ``include/magent_runtime_api.h``;
 * libraries are opened RTLD_LOCAL and cached per path, so two engines can coexist in one process.

There is no CPU fallback: if the CUDA library is missing, loading raises.
"""
from __future__ import annotations

import ctypes
import os
import threading

_c_int_p = ctypes.POINTER(ctypes.c_int)
_c_float_p = ctypes.POINTER(ctypes.c_float)
_vp = ctypes.c_void_p

# name -> argtypes (all return int).  Pointer arguments that the reference wrapper sometimes fills
# with a literal 0 are declared void* so ``0``/``None`` are accepted.
ABI_SIGNATURES = {
    # general environment (reference: src/runtime_api.h:20-36)
    "env_new_game": [ctypes.POINTER(_vp), ctypes.c_char_p],
    "env_delete_game": [_vp],
    "env_config_game": [_vp, ctypes.c_char_p, _vp],
    "env_reset": [_vp],
    "env_get_observation": [_vp, ctypes.c_int, ctypes.POINTER(_vp)],
    "env_set_action": [_vp, ctypes.c_int, _vp],
    "env_step": [_vp, _c_int_p],
    "env_get_reward": [_vp, ctypes.c_int, _vp],
    "env_get_info": [_vp, ctypes.c_int, ctypes.c_char_p, _vp],
    "env_render": [_vp],
    "env_render_next_file": [_vp],
    # gridworld specials (reference: src/runtime_api.h:41-55)
    "gridworld_register_agent_type": [_vp, ctypes.c_char_p, ctypes.c_int,
                                      ctypes.POINTER(ctypes.c_char_p), _c_float_p],
    "gridworld_new_group": [_vp, ctypes.c_char_p, _c_int_p],
    "gridworld_add_agents": [_vp, ctypes.c_int, ctypes.c_int, ctypes.c_char_p, _vp, _vp, _vp],
    "gridworld_clear_dead": [_vp],
    "gridworld_set_goal": [_vp, ctypes.c_int, ctypes.c_char_p, _vp],
    "gridworld_define_agent_symbol": [_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int],
    "gridworld_define_event_node": [_vp, ctypes.c_int, ctypes.c_int, _c_int_p, ctypes.c_int],
    "gridworld_add_reward_rule": [_vp, ctypes.c_int, _c_int_p, _c_float_p, ctypes.c_int,
                                  ctypes.c_bool, ctypes.c_bool],
    # the second game behind the same ABI (reference: src/runtime_api.h:60-61); out of scope for
    # the B200 engine, exported so a drop-in .so resolves every symbol.
    "discrete_snake_clear_dead": [_vp],
    "discrete_snake_add_object": [_vp, ctypes.c_int, ctypes.c_int, ctypes.c_char_p, _vp],
}

# B200 extensions (include/magent_b200_ext.h); absent from the reference library.
EXT_SIGNATURES = {
    "magent_b200_version": ([], ctypes.c_int),
    "magent_b200_host_alloc": ([ctypes.c_size_t], _vp),
    "magent_b200_host_free": ([_vp], ctypes.c_int),
    "magent_b200_device_count": ([], ctypes.c_int),
    "magent_b200_sync": ([_vp], ctypes.c_int),
    "magent_b200_select_arena": ([_vp, ctypes.c_int], ctypes.c_int),
    "magent_b200_random_actions": ([_vp, ctypes.c_int, _vp, ctypes.c_ulonglong], ctypes.c_int),
    "magent_b200_get_action_mask": ([_vp, ctypes.c_int, _vp], ctypes.c_int),
    "magent_b200_random_legal_actions": ([_vp, ctypes.c_int, ctypes.c_ulonglong], ctypes.c_int),
    "magent_b200_get_mean_action": ([_vp, ctypes.c_int, ctypes.c_int, _vp, _vp], ctypes.c_int),
    "magent_b200_get_neighbours": ([_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp, _vp, _vp], ctypes.c_int),
    "magent_b200_get_slots": ([_vp, ctypes.c_int, _vp, _vp], ctypes.c_int),
    "magent_b200_get_observation_slots": ([_vp, ctypes.c_int, ctypes.POINTER(_vp), ctypes.c_int], ctypes.c_int),
    "magent_b200_set_action_slots": ([_vp, ctypes.c_int, _vp], ctypes.c_int),
    "magent_b200_get_reward_slots": ([_vp, ctypes.c_int, _vp, _vp], ctypes.c_int),
    "magent_b200_get_action_mask_slots": ([_vp, ctypes.c_int, _vp], ctypes.c_int),
    "magent_b200_get_mean_action_slots": ([_vp, ctypes.c_int, ctypes.c_int, _vp, _vp], ctypes.c_int),
    "magent_b200_get_neighbours_slots": ([_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp, _vp, _vp], ctypes.c_int),
    "magent_b200_rule_actions": ([_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_ulonglong], ctypes.c_int),
    "magent_b200_get_rule_actions": ([_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_ulonglong, _vp], ctypes.c_int),
    "magent_b200_get_rule_actions_slots": ([_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_ulonglong, _vp],
                                           ctypes.c_int),
    "magent_b200_get_observation_f16": ([_vp, ctypes.c_int, ctypes.POINTER(_vp)], ctypes.c_int),
    "magent_b200_get_global_state": ([_vp, _vp, ctypes.c_int], ctypes.c_int),
    "magent_b200_snapshot_arenas": ([_vp], ctypes.c_int),
    "magent_b200_free_snapshot": ([_vp, ctypes.c_int], ctypes.c_int),
    "magent_b200_restore_arenas": ([_vp, ctypes.c_int, _vp, ctypes.c_int], ctypes.c_int),
    "magent_b200_replay_new": ([_vp, _vp, ctypes.c_int, ctypes.c_int], ctypes.c_int),
    "magent_b200_replay_record": ([_vp, ctypes.c_int], ctypes.c_int),
    "magent_b200_replay_write": ([_vp, ctypes.c_int, ctypes.c_char_p, _vp], ctypes.c_int),
    "magent_b200_replay_free": ([_vp, ctypes.c_int], ctypes.c_int),
    "magent_b200_get_arena_done": ([_vp, _vp], ctypes.c_int),
    "magent_b200_get_counters": ([_vp, ctypes.POINTER(ctypes.c_longlong), ctypes.c_int], ctypes.c_int),
    "magent_b200_last_error": ([], ctypes.c_char_p),
    "magent_b200_set_profiling": ([_vp, ctypes.c_int], ctypes.c_int),
    "magent_b200_get_profile": ([_vp, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_longlong)], ctypes.c_int),
    "magent_b200_stream": ([_vp], _vp),
    "magent_b200_graph_begin": ([_vp], ctypes.c_int),
    "magent_b200_graph_end": ([_vp], ctypes.c_int),
    "magent_b200_graph_launch": ([_vp, ctypes.c_int, ctypes.c_int], ctypes.c_int),
    "magent_b200_get_io_stats": ([_vp, ctypes.POINTER(ctypes.c_longlong), ctypes.c_int], ctypes.c_int),
    "magent_b200_host_threads": ([], ctypes.c_int),
    "magent_b200_numa_nodes": ([], ctypes.c_int),
    "magent_b200_set_host_threads": ([ctypes.c_int], ctypes.c_int),
    "magent_b200_launch_count": ([], ctypes.c_longlong),
}

_HERE = os.path.dirname(os.path.abspath(__file__))
DEFAULT_LIB = os.path.join(_HERE, "lib", "libmagent.so")

_cache = {}
_cache_lock = threading.Lock()


class EngineLibrary:
    """A dlopen'ed ABI library plus feature flags."""

    def __init__(self, path):
        self.path = os.path.abspath(path)
        if not os.path.exists(self.path):
            raise OSError(
                "engine library %s not found; build it with `python -c 'import __graft_entry__ as g; "
                "g.build()'` (there is no CPU fallback)" % self.path)
        self.cdll = ctypes.CDLL(self.path, mode=ctypes.RTLD_LOCAL)
        for name, argtypes in ABI_SIGNATURES.items():
            fn = getattr(self.cdll, name)       # AttributeError => not a drop-in library
            fn.argtypes = argtypes
            fn.restype = ctypes.c_int
            setattr(self, name, fn)
        self.is_b200 = hasattr(self.cdll, "magent_b200_version")
        if self.is_b200:
            for name, (argtypes, restype) in EXT_SIGNATURES.items():
                fn = getattr(self.cdll, name)
                fn.argtypes = argtypes
                fn.restype = restype
                setattr(self, name, fn)

    def __repr__(self):
        return "EngineLibrary(%r, b200=%s)" % (self.path, self.is_b200)


def load_library(path=None):
    """Open (or fetch from cache) the engine library at ``path``.

    Resolution order: explicit ``path`` > ``$MAGENT_B200_LIB`` > in-tree build product.
    """
    if isinstance(path, EngineLibrary):
        return path
    if path is None:
        path = os.environ.get("MAGENT_B200_LIB", DEFAULT_LIB)
    path = os.path.abspath(path)
    with _cache_lock:
        lib = _cache.get(path)
        if lib is None:
            lib = _cache[path] = EngineLibrary(path)
        return lib


def as_float_c_array(buf):
    """numpy float32 array -> float* (reference: python/magent/c_lib.py:25-27)."""
    return buf.ctypes.data_as(_c_float_p)


def as_int32_c_array(buf):
    """numpy int32 array -> int* (reference: python/magent/c_lib.py:30-32)."""
    return buf.ctypes.data_as(_c_int_p)


def as_bool_c_array(buf):
    """numpy bool array -> bool* (reference: python/magent/c_lib.py:35-37)."""
    return buf.ctypes.data_as(ctypes.POINTER(ctypes.c_bool))
