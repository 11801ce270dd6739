"""Host-side mirror of the reference ``magent.gridworld`` surface for the B200 engine.

Same public names, argument meaning and return types as the reference wrapper
(reference: python/magent/gridworld.py:14-800) so that ``examples/train_{battle,pursuit,gather}.py``
run unchanged, but written against the typed ABI table in :mod:`magent_b200.c_lib`:

* the library is per-instance (``_lib=`` keyword or ``$MAGENT_B200_LIB``), which lets the parity
  tests drive the compiled reference engine and the CUDA engine with one and the same host code;
* observation / reward / info buffers are cached per group and, when the library is the B200
  engine, live in page-locked host memory handed out by ``magent_b200_host_alloc`` so the
  device->host copy behind ``env_get_observation`` runs at PCIe speed;
* B200 extensions: ``_num_arenas`` (independent arenas batched behind one handle; every group is
  presented as the concatenation over arenas), device-pointer observation (``get_observation_torch``),
  on-device random actions for throughput runs, event counters.

Reserved constructor keywords start with an underscore so they can never collide with the keyword
arguments forwarded to a built-in config's ``get_config``.
"""
from __future__ import annotations

import ctypes
import importlib
import os

import numpy as np

from .c_lib import load_library, as_float_c_array, as_int32_c_array
from .environment import Environment


def _cint(v):
    return ctypes.byref(ctypes.c_int(int(v)))


def _dptr(t):
    """a tensor's data for the ABI; None (NULL) for None or an empty tensor, which has nothing to receive"""
    return None if t is None or t.numel() == 0 else ctypes.c_void_p(t.data_ptr())


def _check_cuda_out(t, what, dtypes, rows=None, tail=(), shape=None, align=1, optional=False):
    """raise ValueError unless `t` is a contiguous CUDA tensor of one of `dtypes`, `align`-byte aligned, of exactly
    `shape` or else of shape (r,) + tail with r >= rows.  optional: None is accepted too."""
    import torch
    if t is None and optional:
        return
    ok = (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype in dtypes and t.is_contiguous() and
          t.data_ptr() % align == 0)
    if ok:
        s = tuple(t.shape)
        ok = s == tuple(shape) if shape is not None else (len(s) == 1 + len(tail) and s[0] >= rows and s[1:] == tail)
    if not ok:
        want = (str(tuple(shape)) if shape is not None else
                "(rows%s) with at least %d rows" % ("".join(", %d" % d for d in tail) or ",", rows))
        raise ValueError("%s must be a contiguous%s CUDA tensor of dtype %s and shape %s" % (
            what, ", %d-byte aligned" % align if align > 1 else "", " or ".join(map(str, dtypes)), want))


def _out_tuple(out, parts):
    """a caller's `out` as one entry per output part (see GridWorld._outputs): the tensor itself for one part, else a
    tuple of tensors in which None may stand for optional parts, not for all"""
    if len(parts) == 1:
        return (out,)
    if not isinstance(out, (tuple, list)) or len(out) != len(parts) or all(t is None for t in out):
        raise ValueError("out must be a (%s) tuple of CUDA tensors, not all None" % ", ".join(p[0] for p in parts))
    return tuple(out)


class _HostBlock:
    """A growable host buffer; page-locked when the engine offers an allocator."""

    def __init__(self, lib):
        self._lib = lib
        self._ptr = None
        self._raw = None
        self._cap = 0

    def view(self, shape, dtype):
        dtype = np.dtype(dtype)
        nbytes = int(np.prod(shape, dtype=np.int64)) * dtype.itemsize
        if nbytes > self._cap or self._raw is None:
            self._grow(max(nbytes, 64))
        return self._raw[:nbytes].view(dtype).reshape(shape)

    def _grow(self, nbytes):
        self.release()
        # populations only shrink between resets: little slack for the big observation buffers (which a multi-socket host
        # splits evenly over its NUMA nodes), room to grow for the small ones
        cap = int(nbytes * (1.02 if nbytes >= (64 << 20) else 1.25)) + 64
        if self._lib.is_b200:
            ptr = self._lib.magent_b200_host_alloc(cap)
            if ptr:
                self._ptr = ptr
                self._raw = np.ctypeslib.as_array(
                    ctypes.cast(ptr, ctypes.POINTER(ctypes.c_uint8)), shape=(cap,))
                self._cap = cap
                return
        self._raw = np.empty((cap,), dtype=np.uint8)
        self._cap = cap

    def release(self):
        if self._ptr is not None:
            self._lib.magent_b200_host_free(self._ptr)
        self._ptr = None
        self._raw = None
        self._cap = 0


class GridWorld(Environment):
    """The grid-world environment (reference: python/magent/gridworld.py:14-566)."""

    OBS_INDEX_VIEW = 0
    OBS_INDEX_HP = 1

    # global keys accepted by env_config_game and the C type behind the void*
    # (reference: python/magent/gridworld.py:46-52, src/gridworld/GridWorld.cc:120-149)
    _CONFIG_TYPES = {
        "map_width": int, "map_height": int,
        "food_mode": bool, "turn_mode": bool, "minimap_mode": bool,
        "revive_mode": bool, "goal_mode": bool,
        "embedding_size": int,
        "render_dir": str,
    }

    def __init__(self, config, **kwargs):
        Environment.__init__(self)
        self._lib = load_library(kwargs.pop("_lib", None))
        self.num_arenas = int(kwargs.pop("_num_arenas", 1))
        device = kwargs.pop("_device", None)
        host_path = kwargs.pop("_host_path", None)      # None: engine default (wire); "dense": dense records over PCIe
        obs_launch = kwargs.pop("_obs_launch", None)    # (grid, chunk, tile) of the observation render; 0 = automatic
        self.game = None

        if isinstance(config, str):
            try:
                module = importlib.import_module("magent.builtin.config." + config)
            except ImportError:
                module = importlib.import_module(__package__ + ".builtin.config." + config)
            try:
                config = getattr(module, "get_config")(**kwargs)
            except AttributeError:
                raise BaseException('unknown built-in game "' + config + '"')
        self.config = config

        L = self._lib
        game = ctypes.c_void_p()
        rc = L.env_new_game(ctypes.byref(game), b"GridWorld")
        if rc != 0 or not game.value:
            why = L.magent_b200_last_error().decode() if L.is_b200 else "env_new_game failed"
            raise RuntimeError("cannot create the GridWorld engine: " + why)
        self.game = game

        # extension keys go first: they size the arena batch before anything else is configured
        if self.num_arenas != 1 or device is not None:
            if not L.is_b200:
                raise ValueError("_num_arenas/_device need the B200 engine library")
            if device is not None:
                L.env_config_game(game, b"device_id", _cint(device))
            L.env_config_game(game, b"num_arenas", _cint(self.num_arenas))
        if host_path is not None:
            if not L.is_b200:
                raise ValueError("_host_path needs the B200 engine library")
            # "dense": dense records over PCIe; "wire": wire records + host expansion whatever the size; default: wire for
            # observations of 16 MB and more, dense below
            L.env_config_game(game, b"host_path", _cint({"dense": 0, "wire": 2, "auto": 1}[host_path]))
        if obs_launch is not None:
            if not L.is_b200:
                raise ValueError("_obs_launch needs the B200 engine library")
            self._set_obs_launch(*obs_launch)

        for key, value in config.config_dict.items():
            kind = self._CONFIG_TYPES[key]
            name = key.encode("ascii")
            if kind is int:
                L.env_config_game(game, name, _cint(value))
            elif kind is bool:
                L.env_config_game(game, name, ctypes.byref(ctypes.c_bool(bool(value))))
            elif kind is str:
                text = value if isinstance(value, bytes) else str(value).encode("ascii")
                L.env_config_game(game, name, ctypes.cast(ctypes.c_char_p(text), ctypes.c_void_p))

        for name, attrs in config.agent_type_dict.items():
            flat = self._flatten_type(attrs)
            n = len(flat)
            keys = (ctypes.c_char_p * n)(*[k.encode("ascii") for k in flat])
            vals = (ctypes.c_float * n)(*[float(v) for v in flat.values()])
            L.gridworld_register_agent_type(game, name.encode("ascii"), n, keys, vals)

        self._serialize_event_exp(config)

        self.group_handles = []
        for type_name in config.groups:
            h = ctypes.c_int32()
            L.gridworld_new_group(game, type_name.encode("ascii"),
                                  ctypes.cast(ctypes.byref(h), ctypes.POINTER(ctypes.c_int)))
            self.group_handles.append(h)

        self._init_obs_buf()

        self.view_space, self.feature_space, self.action_space = {}, {}, {}
        tmp = np.empty((3,), dtype=np.int32)
        for h in self.group_handles:
            L.env_get_info(game, h.value, b"view_space", tmp.ctypes.data)
            self.view_space[h.value] = (int(tmp[0]), int(tmp[1]), int(tmp[2]))
            L.env_get_info(game, h.value, b"feature_space", tmp.ctypes.data)
            self.feature_space[h.value] = (int(tmp[0]),)
            L.env_get_info(game, h.value, b"action_space", tmp.ctypes.data)
            self.action_space[h.value] = (int(tmp[0]),)

    @staticmethod
    def _flatten_type(attrs):
        """Expand Range objects into radius/angle scalars
        (reference: python/magent/gridworld.py:69-80)."""
        flat = {}
        for key, val in attrs.items():
            if key == "view_range":
                flat["view_radius"], flat["view_angle"] = val.radius, val.angle
            elif key == "attack_range":
                flat["attack_radius"], flat["attack_angle"] = val.radius, val.angle
            else:
                flat[key] = val
        return flat

    @staticmethod
    def _hv(handle):
        return handle.value if hasattr(handle, "value") else int(handle)

    # ------------------------------------------------------------------ episode setup
    def reset(self):
        """reset environment (reference: gridworld.py:117-119)"""
        self._lib.env_reset(self.game)

    def add_walls(self, method, **kwargs):
        """add walls; ``method`` in random/custom/fill (reference: gridworld.py:121-141)"""
        kwargs["dir"] = 0
        self.add_agents(-1, method, **kwargs)

    def new_group(self, name):
        """register a new group (reference: gridworld.py:144-148)"""
        h = ctypes.c_int32()
        self._lib.gridworld_new_group(self.game, name.encode("ascii"),
                                      ctypes.cast(ctypes.byref(h), ctypes.POINTER(ctypes.c_int)))
        return h

    def add_agents(self, handle, method, **kwargs):
        """add agents (or walls when handle == -1) (reference: gridworld.py:150-200)

        method="random": kwargs["n"]; "custom": kwargs["pos"] = [(x, y[, dir]), ...];
        "fill": kwargs["pos"]=(x, y), kwargs["size"]=(w, h)[, kwargs["dir"]].
        """
        L, g = self._lib, self._hv(handle)
        if method == "random":
            L.gridworld_add_agents(self.game, g, int(kwargs["n"]), b"random", None, None, None)
        elif method == "custom":
            pos = np.asarray(kwargs["pos"], dtype=np.int32)
            if pos.size == 0:
                return
            n = pos.shape[0]
            xs = np.ascontiguousarray(pos[:, 0])
            ys = np.ascontiguousarray(pos[:, 1])
            dirs = (np.ascontiguousarray(pos[:, 2]) if pos.shape[1] == 3
                    else np.zeros((n,), dtype=np.int32))
            L.gridworld_add_agents(self.game, g, n, b"custom",
                                   xs.ctypes.data, ys.ctypes.data, dirs.ctypes.data)
        elif method == "fill":
            x, y = kwargs["pos"][0], kwargs["pos"][1]
            w, h = kwargs["size"][0], kwargs["size"][1]
            d = kwargs.get("dir", 0)
            bind = np.array([x, y, w, h, d], dtype=np.int32)
            L.gridworld_add_agents(self.game, g, 0, b"fill", bind.ctypes.data, None, None)
        elif method == "maze":
            raise NotImplementedError("maze placement is not implemented by the engine "
                                      "(reference: GridWorld.cc:215-217 raises FATAL as well)")
        else:
            print("Unknown type of position")
            exit(-1)

    # ------------------------------------------------------------------ run
    def _init_obs_buf(self):
        self.obs_bufs = [{}, {}, {}, {}]       # view, feature (reference); f16 view, f16 feature (extension)
        self._blocks = {}

    def _host_view(self, key, shape, dtype):
        """the cached receive buffer `key` as an array of `shape`: valid until the next call with the same key"""
        block = self._blocks.get(key)
        if block is None:
            block = self._blocks[key] = _HostBlock(self._lib)
        return block.view(shape, dtype)

    def _get_obs_buf(self, group, key, shape, dtype):
        """cached receive buffer, resized in place like the reference (gridworld.py:203-213)"""
        buf = self.obs_bufs[key][group] = self._host_view((group, key), shape, dtype)
        return buf

    def get_observation(self, handle):
        """(views, features) of a whole group (reference: gridworld.py:221-248)

        views: float32 (n, view_h, view_w, n_channel); features: float32 (n, feature_size).
        The arrays are the engine's cached receive buffers: valid until the next call.
        """
        g = self._hv(handle)
        n = self.get_num(handle)
        view = self._get_obs_buf(g, self.OBS_INDEX_VIEW, (n,) + self.view_space[g], np.float32)
        feat = self._get_obs_buf(g, self.OBS_INDEX_HP, (n,) + self.feature_space[g], np.float32)
        bufs = (ctypes.c_void_p * 2)(view.ctypes.data, feat.ctypes.data)
        self._lib.env_get_observation(self.game, g, bufs)
        return view, feat

    def set_action(self, handle, actions):
        """actions: int32 numpy array of length get_num(handle) (reference: gridworld.py:250-261)"""
        assert isinstance(actions, np.ndarray)
        assert actions.dtype == np.int32
        actions = np.ascontiguousarray(actions)
        self._lib.env_set_action(self.game, self._hv(handle), actions.ctypes.data)

    def step(self):
        """simulate one step; returns done (reference: gridworld.py:263-273)"""
        done = ctypes.c_int(0)
        self._lib.env_step(self.game, ctypes.byref(done))
        return bool(done.value)

    def get_reward(self, handle):
        """float32 rewards of a group (reference: gridworld.py:275-287)"""
        n = self.get_num(handle)
        buf = np.empty((n,), dtype=np.float32)
        self._lib.env_get_reward(self.game, self._hv(handle), buf.ctypes.data)
        return buf

    def clear_dead(self):
        """remove dead agents; call after step() (reference: gridworld.py:289-293)"""
        self._lib.gridworld_clear_dead(self.game)

    # ------------------------------------------------------------------ info
    def get_handles(self):
        return self.group_handles

    def _info(self, handle, name, buf):
        self._lib.env_get_info(self.game, self._hv(handle), name, buf.ctypes.data)
        return buf

    def get_num(self, handle):
        num = ctypes.c_int(0)
        self._lib.env_get_info(self.game, self._hv(handle), b"num",
                               ctypes.cast(ctypes.byref(num), ctypes.c_void_p))
        return num.value

    def get_action_space(self, handle):
        return self.action_space[self._hv(handle)]

    def get_view_space(self, handle):
        return self.view_space[self._hv(handle)]

    def get_feature_space(self, handle):
        return self.feature_space[self._hv(handle)]

    def get_agent_id(self, handle):
        """int32 ids (reference: gridworld.py:333-345)"""
        return self._info(handle, b"id", np.empty((self.get_num(handle),), dtype=np.int32))

    def get_alive(self, handle):
        """bool alive flags (reference: gridworld.py:347-359)"""
        return self._info(handle, b"alive", np.empty((self.get_num(handle),), dtype=np.bool_))

    def get_pos(self, handle):
        """int32 (n, 2) positions (reference: gridworld.py:361-373)"""
        return self._info(handle, b"pos", np.empty((self.get_num(handle), 2), dtype=np.int32))

    def get_mean_info(self, handle):
        """deprecated (reference: gridworld.py:375-380)"""
        n_act = self.action_space[self._hv(handle)][0]
        return self._info(handle, b"mean_info", np.empty(2 + n_act, dtype=np.float32))

    def get_view2attack(self, handle):
        """(attack_base, view-shaped int32 map of attack action numbers, -1 elsewhere)
        (reference: gridworld.py:382-399)"""
        size = self.get_view_space(handle)[0:2]
        buf = self._info(handle, b"view2attack", np.empty(size, dtype=np.int32))
        base = ctypes.c_int(0)
        self._lib.env_get_info(self.game, self._hv(handle), b"attack_base",
                               ctypes.cast(ctypes.byref(base), ctypes.c_void_p))
        return base.value, buf

    def get_global_minimap(self, height, width):
        """(height, width, n_group) float32 density maps (reference: gridworld.py:401-420)"""
        buf = np.empty((height, width, len(self.group_handles)), dtype=np.float32)
        buf[0, 0, 0] = height
        buf[0, 0, 1] = width
        self._lib.env_get_info(self.game, -1, b"global_minimap", buf.ctypes.data)
        return buf

    def set_seed(self, seed):
        """seed the engine RNG (reference: gridworld.py:422-424)"""
        self._lib.env_config_game(self.game, b"seed", _cint(seed))

    # ------------------------------------------------------------------ render
    def set_render_dir(self, name):
        if not os.path.exists(name):
            os.mkdir(name)
        text = name.encode("ascii")
        self._lib.env_config_game(self.game, b"render_dir",
                                  ctypes.cast(ctypes.c_char_p(text), ctypes.c_void_p))

    def render(self):
        self._lib.env_render(self.game)

    def _get_groups_info(self):
        buf = np.empty((len(self.group_handles), 5), dtype=np.int32)
        self._lib.env_get_info(self.game, -1, b"groups_info", buf.ctypes.data)
        return buf

    def _get_walls_info(self):
        buf = np.empty((100 * 100, 2), dtype=np.int32)
        self._lib.env_get_info(self.game, -1, b"walls_info", buf.ctypes.data)
        n = buf[0, 0]
        return buf[1:1 + n]

    def _get_render_info(self, x_range, y_range):
        n = sum(self.get_num(h) for h in self.group_handles)
        buf = np.empty((n + 1, 4), dtype=np.int32)
        buf[0] = x_range[0], y_range[0], x_range[1], y_range[1]
        self._lib.env_get_info(self.game, -1, b"render_window_info", buf.ctypes.data)
        agent_ct, attack_ct = buf[0][0], buf[0][1]
        agent_info = {row[0]: [row[1], row[2], row[3]] for row in buf[1:1 + agent_ct]}
        events = np.empty((attack_ct, 3), dtype=np.int32)
        self._lib.env_get_info(self.game, -1, b"attack_event", events.ctypes.data)
        return agent_info, events

    def __del__(self):
        game, self.game = getattr(self, "game", None), None
        if game is not None:
            try:
                for block in getattr(self, "_blocks", {}).values():
                    block.release()
                self._lib.env_delete_game(game)
            except Exception:       # interpreter shutdown
                pass

    # ------------------------------------------------------------------ special rule
    def set_goal(self, handle, method, *args, **kwargs):
        """deprecated (reference: gridworld.py:485-490)"""
        if method == "random":
            self._lib.gridworld_set_goal(self.game, self._hv(handle), b"random", None)
        else:
            raise NotImplementedError

    # ------------------------------------------------------------------ B200 extensions
    def get_arena_nums(self, handle):
        """per-arena agent counts of a group (extension; int32 [num_arenas])"""
        buf = np.empty((self.num_arenas,), dtype=np.int32)
        return self._info(handle, b"arena_num", buf)

    def get_arena_done(self):
        """per-arena done flags of the last step (extension; int32 [num_arenas])"""
        buf = np.empty((self.num_arenas,), dtype=np.int32)
        self._lib.env_get_info(self.game, -1, b"arena_done", buf.ctypes.data)
        return buf

    def select_arena(self, arena):
        """route subsequent setup calls (add_agents/add_walls/set_seed) to one arena; -1 = all"""
        self._lib.magent_b200_select_arena(self.game, int(arena))

    def get_observation_torch(self, handle, out=None, dtype=None):
        """observation written straight into CUDA tensors through the same ABI call
        (device pointers are detected by the engine; no PCIe traffic).

        dtype: torch.float32 (default, the reference layout) or torch.float16 (compact hand-off: every element
        is the float32 value rounded to nearest-even; half the bytes).
        out: a caller-owned (view, feature) pair of contiguous CUDA tensors of one of those dtypes, (rows,) + view_space
        and (rows,) + feature_space with at least get_num(handle) rows; returned whole."""
        import torch
        g = self._hv(handle)
        n = self.get_num(handle)
        if out is None:
            view, feat = (torch.empty((n,) + tail, dtype=getattr(torch, dtypes[0]), device="cuda")
                          for _name, dtypes, tail, _opt in self._obs_parts(g, dtype))
        else:
            # at least get_num rows: the engine writes that many records through device pointers
            view, feat = _out_tuple(out, self._obs_parts(g))
            _check_cuda_out(view, "view", (torch.float32, torch.float16), rows=n, tail=self.view_space[g])
            _check_cuda_out(feat, "feature", (view.dtype,), rows=n, tail=self.feature_space[g])
        bufs = (ctypes.c_void_p * 2)(view.data_ptr(), feat.data_ptr())
        if view.dtype == torch.float16:
            self._lib.magent_b200_get_observation_f16(self.game, g, bufs)
        else:
            self._lib.env_get_observation(self.game, g, bufs)
        return view, feat

    def get_observation_f16(self, handle):
        """(views, features) as float16 numpy arrays (compact hand-off; see get_observation for the layout)"""
        g = self._hv(handle)
        n = self.get_num(handle)
        view = self._get_obs_buf(g, 2, (n,) + self.view_space[g], np.float16)
        feat = self._get_obs_buf(g, 3, (n,) + self.feature_space[g], np.float16)
        bufs = (ctypes.c_void_p * 2)(view.ctypes.data, feat.ctypes.data)
        self._lib.magent_b200_get_observation_f16(self.game, g, bufs)
        return view, feat

    def get_state_space(self):
        """(H, W, C) of one arena's global state (extension; see get_global_state)"""
        buf = np.empty((3,), dtype=np.int32)
        self._lib.env_get_info(self.game, -1, b"state_space", buf.ctypes.data)
        return int(buf[0]), int(buf[1]), int(buf[2])

    def get_global_state(self):
        """whole-map global state of every arena (extension): float32 (num_arenas, H, W, C).

        Per map cell: channel 0 wall, channel 1 food (food_mode only), then per group g in absolute order
        base + 2g presence and base + 2g + 1 hp / max_hp (base = 1 + food_mode); 0 elsewhere.  Every value equals
        the one a view covering the cell shows.  The array is a cached receive buffer: valid until the next call."""
        buf = self._host_view("state", (self.num_arenas,) + self.get_state_space(), np.float32)
        self._lib.magent_b200_get_global_state(self.game, buf.ctypes.data, 0)
        return buf

    def get_global_state_torch(self, out=None, dtype=None):
        """the global state (see get_global_state) written straight into a CUDA tensor (num_arenas, H, W, C).

        dtype: torch.float32 (default) or torch.float16 (every element the float32 value rounded to nearest-even).
        out: a caller-owned contiguous CUDA tensor of that shape, 16-byte aligned; needed to record the call into a
        CUDA graph (capture_graph), since the call then allocates nothing."""
        import torch
        shape = (self.num_arenas,) + self.get_state_space()
        if out is None:
            out = torch.empty(shape, dtype=torch.float32 if dtype is None else dtype, device="cuda")
        elif dtype is not None and out.dtype != dtype:
            raise ValueError("out has dtype %s, not %s" % (out.dtype, dtype))
        _check_cuda_out(out, "out", (torch.float32, torch.float16), shape=shape, align=16)
        self._lib.magent_b200_get_global_state(self.game, ctypes.c_void_p(out.data_ptr()),
                                               1 if out.dtype == torch.float16 else 0)
        return out

    # ---- reset pool: restart finished arenas from device-resident snapshots
    def _check(self, rc, what):
        if rc < 0:
            raise RuntimeError("%s refused: %s" % (what, self._lib.magent_b200_last_error().decode()))
        return rc

    def snapshot_arenas(self):
        """copy the state of every arena into a new snapshot in device memory; returns its id"""
        return self._check(self._lib.magent_b200_snapshot_arenas(self.game), "snapshot_arenas")

    def free_snapshot(self, snapshot):
        self._check(self._lib.magent_b200_free_snapshot(self.game, int(snapshot)), "free_snapshot")

    def restore_arenas(self, snapshot, src=None, keep_rng=False):
        """make arena a exactly arena src[a] of the snapshot (src[a] = -1: leave it alone).

        src: None (every arena whose last step reported done takes its own snapshot arena, decided on the device), an
        int32 numpy array or an int32 CUDA tensor of length num_arenas (passed as a device pointer: nothing waits for the
        host, and the call can be recorded into a CUDA graph).  keep_rng: restored arenas keep their own RNG stream."""
        if src is None:
            ptr = None
        elif isinstance(src, np.ndarray):
            if src.dtype != np.int32 or src.shape != (self.num_arenas,):
                raise ValueError("src must be an int32 array of shape (%d,)" % self.num_arenas)
            src = np.ascontiguousarray(src)
            ptr = src.ctypes.data
        else:
            import torch
            _check_cuda_out(src, "src (when not an int32 numpy array)", (torch.int32,), shape=(self.num_arenas,))
            ptr = src.data_ptr()
        self._check(self._lib.magent_b200_restore_arenas(self.game, int(snapshot), ptr, 1 if keep_rng else 0),
                    "restore_arenas")

    # ---- replay recorder: watch chosen arenas of a device-resident loop in the reference viewer's format
    def new_replay(self, arenas, max_frames):
        """a recorder of the listed arenas with room for max_frames frames on the device; returns its id.  Make it
        before capturing any CUDA graph: steps captured without a live recorder record no attack events."""
        arr = np.ascontiguousarray(np.asarray(arenas, dtype=np.int32).reshape(-1))
        return self._check(self._lib.magent_b200_replay_new(self.game, arr.ctypes.data, int(arr.size), int(max_frames)),
                           "new_replay")

    def record_replay(self, replay):
        """append one frame of every arena of the recorder, the frame render() would write for it; waits for nothing
        and can be recorded into a CUDA graph (capture_graph)"""
        self._check(self._lib.magent_b200_replay_record(self.game, int(replay)), "record_replay")

    def write_replay(self, replay, directory):
        """write the buffered frames as directory/arena_<a>/config.json and video_<k>.txt and empty the buffer;
        returns (frames written per arena, frames dropped for want of room since the last write)"""
        dropped = ctypes.c_longlong(0)
        n = self._check(self._lib.magent_b200_replay_write(self.game, int(replay), os.fsencode(directory),
                                                           ctypes.addressof(dropped)), "write_replay")
        return n, int(dropped.value)

    def free_replay(self, replay):
        self._check(self._lib.magent_b200_replay_free(self.game, int(replay)), "free_replay")

    def get_arena_done_torch(self, out=None):
        """per-arena done flags of the last step into an int32 CUDA tensor (num_arenas,); nothing waits for the host"""
        import torch
        if out is None:
            out = torch.empty((self.num_arenas,), dtype=torch.int32, device="cuda")
        _check_cuda_out(out, "out", (torch.int32,), shape=(self.num_arenas,))
        self._check(self._lib.magent_b200_get_arena_done(self.game, out.data_ptr()), "get_arena_done")
        return out

    def get_arena_rng(self):
        """uint32 minstd state of every arena (the "seed" that continues its stream)"""
        buf = np.empty((self.num_arenas,), dtype=np.uint32)
        self._lib.env_get_info(self.game, -1, b"arena_rng", buf.ctypes.data)
        return buf

    def get_num_bound(self, handle):
        """the most records a device-pointer call for this group can write before the counts next settle: the size for
        device buffers of a CUDA graph that restores arenas (see restore_arenas)"""
        buf = np.empty((len(self.group_handles),), dtype=np.int32)
        self._lib.env_get_info(self.game, -1, b"num_bound", buf.ctypes.data)
        return int(buf[self._hv(handle)])

    def set_random_actions(self, handle, seed):
        """uniform random actions generated on the device (throughput runs only)"""
        self._lib.magent_b200_random_actions(self.game, self._hv(handle), None, int(seed))

    # ---- per-agent outputs, in rows (the order of set_action) or in the stable slot layout (see get_slots).  Whether a
    # call reaches the engine with nothing to write (an empty group, S = 0) is each method's own: the engine checks the
    # arguments of any call it gets (groups, k, policy, a kernel's limits), and refuses an empty tensor's NULL data for
    # a part it needs.
    # An output part: (name, its torch dtype names, the first also its numpy dtype and the one allocated, its per-record
    # shape, whether a caller's out may give None for it: passed as NULL, returned as None).
    _RULE_PARTS = (("act", ("int32",), (), False),)
    _REWARD_PARTS = (("reward", ("float32",), (), True), ("status", ("uint8",), (), True))

    def _mask_parts(self, g):
        return (("mask", ("bool", "uint8"), (self.action_space[g][0],), False),)

    def _mean_parts(self, of, slots=False):          # count may be None in the slot-ordered form only
        return (("mean", ("float32",), (self.action_space[of][0],), False), ("count", ("int32",), (), slots))

    @staticmethod
    def _nbr_parts(k):                              # (k, checked, and the parts)
        k = int(k)
        if not 1 <= k <= 32:
            raise ValueError("k must be in [1, 32], got %d" % k)
        return k, (("idx", ("int32",), (k,), False), ("rel", ("int32",), (k, 2), True), ("count", ("int32",), (), True))

    def _obs_parts(self, g, dtype=None):            # float32 or float16, or the one of them `dtype` names
        if dtype is not None and str(dtype) not in ("torch.float32", "torch.float16"):
            raise ValueError("observation dtype must be torch.float32 or torch.float16")
        names = ("float32", "float16") if dtype is None else (str(dtype)[len("torch."):],)
        return (("view", names, self.view_space[g], False), ("feature", names, self.feature_space[g], False))

    def _groups(self, handle, of):                  # `of` is the group itself by default
        g = self._hv(handle)
        return g, g if of is None else self._hv(of)

    def _outputs(self, handle, parts, slots=False, out=None, host=None):
        """(the data of one output call's buffers for the ABI, the results, whether the call has anything to write: the
        first buffer given holds a record).  slots: lead (num_arenas, S) and a caller's tensors of exactly that lead;
        else lead (get_num(handle),), a caller's tensors of at least get_num_bound(handle) rows, the results trimmed to
        the lead.  host: the name of the cached host buffers (numpy) to receive into, valid until the next call with
        that name for the group; else CUDA tensors, new ones or the caller's `out`, checked before anything is done."""
        lead = self._slot_shape(handle) if slots else (self.get_num(handle),)
        if host is not None:
            g = self._hv(handle)
            bufs = [self._host_view((g, host, name), lead + tail, dtypes[0]) for name, dtypes, tail, _ in parts]
            return [b.ctypes.data for b in bufs], tuple(bufs), 0 not in lead
        import torch
        if out is None:
            bufs = [torch.empty(lead + tail, dtype=getattr(torch, dtypes[0]), device="cuda")
                    for _name, dtypes, tail, _opt in parts]
        else:
            bufs = _out_tuple(out, parts)
            bound = None if slots else self.get_num_bound(handle)
            for t, (name, dtypes, tail, optional) in zip(bufs, parts):
                _check_cuda_out(t, name if len(parts) > 1 else "out", tuple(getattr(torch, d) for d in dtypes),
                                rows=bound, tail=tail, shape=lead + tail if slots else None, optional=optional)
        todo = 0 not in next(t for t in bufs if t is not None).shape
        ptrs = [None if t is None else ctypes.c_void_p(t.data_ptr()) for t in bufs]
        return ptrs, tuple(t if slots or t is None else t[:lead[0]] for t in bufs), todo

    def get_action_mask(self, handle):
        """bool (n, n_action): which actions of every agent of the group would succeed if taken alone on the state as it
        is now (include/magent_b200_ext.h magent_b200_get_action_mask has the definition).  Rows are in the order of
        set_action; a dead, un-culled agent's row is all False.  The array is a cached receive buffer: valid until the
        next call."""
        g = self._hv(handle)
        (ptr,), (mask,), _ = self._outputs(handle, self._mask_parts(g), host="mask")
        self._check(self._lib.magent_b200_get_action_mask(self.game, g, ptr), "get_action_mask")
        return mask

    def get_action_mask_torch(self, handle, out=None):
        """the legal-action mask (see get_action_mask) written straight into a CUDA torch.bool tensor (n, n_action):
        logits.masked_fill_(~mask, -inf) before sampling.

        out: a caller-owned contiguous CUDA tensor (rows, n_action), torch.bool or torch.uint8, with at least
        get_num_bound(handle) rows; needed to record the call into a CUDA graph (capture_graph), since the call then
        allocates nothing.  Returns the first get_num(handle) rows as torch.bool."""
        import torch
        g = self._hv(handle)
        (ptr,), (mask,), _ = self._outputs(handle, self._mask_parts(g), out=out)
        self._check(self._lib.magent_b200_get_action_mask(self.game, g, ptr), "get_action_mask")
        return mask.view(torch.bool)

    def set_random_legal_actions(self, handle, seed):
        """set_action with an action drawn uniformly from every agent's legal actions (get_action_mask), on the device:
        the exploration baseline, and a much denser fight than set_random_actions produces"""
        self._check(self._lib.magent_b200_random_legal_actions(self.game, self._hv(handle), int(seed)),
                    "random_legal_actions")

    def get_mean_action(self, handle, of=None):
        """(mean float32 (n, n_action(of)), count int32 (n,)): for every agent of the group, the mean one-hot action of
        the agents of group `of` (default: its own group) that its view shows, and how many those are -- mean-field
        Q-learning's neighbour action (include/magent_b200_ext.h magent_b200_get_mean_action has the definition).  Called
        after step and before the next set_action it gives the previous step's actions.  Rows are in the order of
        set_action.  Both arrays are cached receive buffers: valid until the next call."""
        g, o = self._groups(handle, of)
        ptrs, res, _ = self._outputs(handle, self._mean_parts(o), host="mean")
        self._check(self._lib.magent_b200_get_mean_action(self.game, g, o, *ptrs), "get_mean_action")
        return res

    def get_mean_action_torch(self, handle, of=None, out=None):
        """the mean neighbour action (see get_mean_action) written straight into CUDA tensors: returns (mean float32
        (n, n_action(of)), count int32 (n,)).

        out: a caller-owned pair (mean, count) of contiguous CUDA tensors, float32 (rows, n_action(of)) and int32
        (rows,), with at least get_num_bound(handle) rows each; needed to record the call into a CUDA graph
        (capture_graph), since the call then allocates nothing.  Returns the first get_num(handle) rows of each."""
        g, o = self._groups(handle, of)
        ptrs, res, _ = self._outputs(handle, self._mean_parts(o), out=out)
        self._check(self._lib.magent_b200_get_mean_action(self.game, g, o, *ptrs), "get_mean_action")
        return res

    def get_neighbours(self, handle, k, of=None):
        """(idx int32 (n, k), rel int32 (n, k, 2), count int32 (n,)): for every agent of the group, the first k of the
        agents of group `of` (default: its own group) that its view shows, nearest first -- the neighbour lists of
        graph-convolutional and attention policies (include/magent_b200_ext.h magent_b200_get_neighbours has the
        definition).  idx: their rows in group `of`'s order (get_pos(of), get_observation(of)), rel: the (vy, vx) view
        cell where the observer's own observation shows them, count: how many neighbours it has in all.  Unused slots
        are -1.  Rows are in the order of set_action.  The arrays are cached receive buffers: valid until the next call."""
        g, o = self._groups(handle, of)
        k, parts = self._nbr_parts(k)
        ptrs, res, _ = self._outputs(handle, parts, host="nbr")
        self._check(self._lib.magent_b200_get_neighbours(self.game, g, o, k, *ptrs), "get_neighbours")
        return res

    def get_neighbours_torch(self, handle, k, of=None, out=None):
        """the nearest visible neighbours (see get_neighbours) written straight into CUDA tensors: returns (idx int32
        (n, k), rel int32 (n, k, 2), count int32 (n,)).

        out: a caller-owned triple (idx, rel, count) of contiguous CUDA int32 tensors of shapes (rows, k), (rows, k, 2)
        and (rows,), with at least get_num_bound(handle) rows each; needed to record the call into a CUDA graph
        (capture_graph), since the call then allocates nothing.  rel and count may be None: they are then neither
        computed nor written (without count the kernel stops at the k-th neighbour), and None comes back in their place.
        Returns the first get_num(handle) rows of each."""
        g, o = self._groups(handle, of)
        k, parts = self._nbr_parts(k)
        ptrs, res, todo = self._outputs(handle, parts, out=out)
        if todo:            # no row can be written, and the engine refuses the NULL data of an empty idx
            self._check(self._lib.magent_b200_get_neighbours(self.game, g, o, k, *ptrs), "get_neighbours")
        return res

    def get_slot_space(self, handle):
        """S, the slot space of the group: slots run over [0, S) in every arena (include/magent_b200_ext.h
        magent_b200_get_slots has the definition).  Only reset, add_agents, snapshot_arenas and free_snapshot change it;
        nothing waits for the device."""
        buf = np.empty((len(self.group_handles),), dtype=np.int32)
        self._lib.env_get_info(self.game, -1, b"slot_space", buf.ctypes.data)
        return int(buf[self._hv(handle)])

    def get_slots(self, handle):
        """(row_slot int32 (n,), slot_row int32 (num_arenas, S)): the stable slot of every agent of the group.  An agent's
        slot is the number of agents of its group placed into its arena before it since the last reset; it survives
        clear_dead, and a restored arena's agents keep the slots they have in the snapshot.  row_slot[r] = a * S + slot
        for row r (the order of set_action), a its arena; slot_row[a, slot] = the row of the agent in that slot, -1 when
        the slot is vacant.  Both arrays are cached receive buffers: valid until the next call."""
        g = self._hv(handle)
        n = self.get_num(handle)                 # settles the counts, so the bound below is the call's
        bound = self.get_num_bound(handle)
        S = self.get_slot_space(handle)
        raw = self._host_view((g, "slots"), (bound + self.num_arenas * S,), np.int32)
        row_slot, slot_row = raw[:bound], raw[bound:].reshape(self.num_arenas, S)
        self._check(self._lib.magent_b200_get_slots(self.game, g, row_slot.ctypes.data, slot_row.ctypes.data),
                    "get_slots")
        return row_slot[:n], slot_row

    def get_slots_torch(self, handle, out=None):
        """the stable slots (see get_slots) written straight into CUDA tensors, without waiting for the device: returns
        (row_slot int32 (num_bound,), slot_row int32 (num_arenas, S)).  Entries of row_slot from the device-side count of
        the group on are -1, so it is also the valid-row mask of the group's row-ordered outputs.  Scatter rows into
        slots with x[slot_row.clamp(min=0)] and gather slot-ordered actions back with act_s.view(-1)[row_slot.clamp(min=0)]
        (INTEGRATION.md §4).

        out: a caller-owned pair (row_slot, slot_row) of contiguous CUDA int32 tensors, of shapes (rows,) with at least
        get_num_bound(handle) rows and (num_arenas, get_slot_space(handle)); needed to record the call into a CUDA graph
        (capture_graph), since the call then allocates nothing.  Either may be None: it is then not written, and None comes
        back in its place.  The first get_num_bound(handle) entries of row_slot are written."""
        import torch
        g = self._hv(handle)
        bound = self.get_num_bound(handle)
        S = self.get_slot_space(handle)
        if out is None:
            row_slot = torch.empty((bound,), dtype=torch.int32, device="cuda")
            slot_row = torch.empty((self.num_arenas, S), dtype=torch.int32, device="cuda")
        else:
            if not isinstance(out, (tuple, list)) or len(out) != 2 or (out[0] is None and out[1] is None):
                raise ValueError("out must be a (row_slot, slot_row) pair of CUDA tensors, at most one of them None")
            row_slot, slot_row = out
            _check_cuda_out(row_slot, "row_slot", (torch.int32,), rows=bound, optional=True)
            _check_cuda_out(slot_row, "slot_row", (torch.int32,), shape=(self.num_arenas, S), optional=True)
        if _dptr(row_slot) is None and _dptr(slot_row) is None:
            return row_slot, slot_row
        self._check(self._lib.magent_b200_get_slots(self.game, g, _dptr(row_slot), _dptr(slot_row)), "get_slots")
        return row_slot, slot_row

    def get_observation_slots(self, handle):
        """(views, features) of a whole group in the stable slot layout (see get_slots): float32
        (num_arenas, S) + view_space and (num_arenas, S) + feature_space, S = get_slot_space(handle).  Slot (a, s) holds
        the record get_observation gives the row slot_row[a, s]; a vacant slot is all zeros.  The arrays are cached
        receive buffers: valid until the next call."""
        g = self._hv(handle)
        ptrs, res, todo = self._outputs(handle, self._obs_parts(g), slots=True, host="obs_slots")
        if todo:
            self._check(self._lib.magent_b200_get_observation_slots(self.game, g, (ctypes.c_void_p * 2)(*ptrs), 0),
                        "get_observation_slots")
        return res

    def get_observation_slots_torch(self, handle, out=None, dtype=None):
        """the slot-ordered observation (see get_observation_slots) rendered straight into CUDA tensors, without waiting
        for the device: (view (num_arenas, S) + view_space, feature (num_arenas, S) + feature_space).

        dtype: torch.float32 (default) or torch.float16 (every element the float32 value rounded to nearest-even).
        out: a caller-owned (view, feature) pair of contiguous CUDA tensors of those shapes and one dtype; needed to
        record the call into a CUDA graph (capture_graph), since the call then allocates nothing once a first call has
        run."""
        import torch
        g = self._hv(handle)
        ptrs, (view, feat), todo = self._outputs(handle, self._obs_parts(g, dtype), slots=True, out=out)
        if feat.dtype != view.dtype:
            raise ValueError("view and feature must be of one dtype, not %s and %s" % (view.dtype, feat.dtype))
        if todo:
            self._check(self._lib.magent_b200_get_observation_slots(self.game, g, (ctypes.c_void_p * 2)(*ptrs),
                                                                    1 if view.dtype == torch.float16 else 0),
                        "get_observation_slots")
        return view, feat

    def _slot_shape(self, handle):
        return (self.num_arenas, self.get_slot_space(handle))

    def set_action_slots(self, handle, actions):
        """set_action in the stable slot layout (see get_slots): every agent takes actions[a, s] of its arena and slot;
        vacant slots are never read.  actions: an int32 numpy array (num_arenas, S) or a contiguous CUDA int32 tensor of
        that shape (nothing waits for the device, and the call can be recorded into a CUDA graph).  It counts as the
        group's set_action for the step (include/magent_b200_ext.h magent_b200_set_action_slots has the definition)."""
        g = self._hv(handle)
        shape = self._slot_shape(handle)
        if isinstance(actions, np.ndarray):
            if actions.dtype != np.int32 or actions.shape != shape:
                raise ValueError("actions must be an int32 array of shape %s" % (shape,))
            actions = np.ascontiguousarray(actions)
            ptr = actions.ctypes.data if actions.size else None
        else:
            import torch
            _check_cuda_out(actions, "actions (when not an int32 numpy array)", (torch.int32,), shape=shape)
            ptr = _dptr(actions)
        self._check(self._lib.magent_b200_set_action_slots(self.game, g, ptr), "set_action_slots")

    def get_reward_slots(self, handle):
        """(reward float32 (num_arenas, S), status uint8 (num_arenas, S)) in the stable slot layout: the reward get_reward
        gives the agent in each slot and 0 vacant / 1 alive / 2 dead but not culled yet (between step and clear_dead, 2
        is the per-agent terminal signal); +0.0 and 0 in vacant slots.  Both arrays are cached receive buffers: valid
        until the next call."""
        g = self._hv(handle)
        ptrs, res, todo = self._outputs(handle, self._REWARD_PARTS, slots=True, host="reward_slots")
        if todo:
            self._check(self._lib.magent_b200_get_reward_slots(self.game, g, *ptrs), "get_reward_slots")
        return res

    def get_reward_slots_torch(self, handle, out=None):
        """the slot-ordered reward and status (see get_reward_slots) written straight into CUDA tensors, without waiting
        for the device: (reward float32 (num_arenas, S), status uint8 (num_arenas, S)).

        out: a caller-owned pair (reward, status) of contiguous CUDA tensors of those shapes and dtypes; needed to record
        the call into a CUDA graph (capture_graph), since the call then allocates nothing.  Either may be None: it is
        then not written, and None comes back in its place."""
        g = self._hv(handle)
        ptrs, res, todo = self._outputs(handle, self._REWARD_PARTS, slots=True, out=out)
        if todo:
            self._check(self._lib.magent_b200_get_reward_slots(self.game, g, *ptrs), "get_reward_slots")
        return res

    def get_action_mask_slots(self, handle):
        """bool (num_arenas, S, n_action): the legal-action mask (see get_action_mask) in the stable slot layout; all
        False in vacant slots and for dead, un-culled agents.  The array is a cached receive buffer: valid until the next
        call."""
        g = self._hv(handle)
        (ptr,), (mask,), todo = self._outputs(handle, self._mask_parts(g), slots=True, host="mask_slots")
        if todo:
            self._check(self._lib.magent_b200_get_action_mask_slots(self.game, g, ptr), "get_action_mask_slots")
        return mask

    def get_action_mask_slots_torch(self, handle, out=None):
        """the slot-ordered legal-action mask (see get_action_mask_slots) written straight into a CUDA torch.bool tensor
        (num_arenas, S, n_action), without waiting for the device.

        out: a caller-owned contiguous CUDA tensor of that shape, torch.bool or torch.uint8; needed to record the call
        into a CUDA graph (capture_graph), since the call then allocates nothing once a first call has run."""
        import torch
        g = self._hv(handle)
        (ptr,), (mask,), todo = self._outputs(handle, self._mask_parts(g), slots=True, out=out)
        if todo:
            self._check(self._lib.magent_b200_get_action_mask_slots(self.game, g, ptr), "get_action_mask_slots")
        return mask.view(torch.bool)

    def get_mean_action_slots(self, handle, of=None):
        """(mean float32 (num_arenas, S, n_action(of)), count int32 (num_arenas, S)): the mean neighbour action (see
        get_mean_action) in the stable slot layout (see get_slots); a +0.0 row and count 0 in vacant slots.  Both arrays
        are cached receive buffers: valid until the next call."""
        g, o = self._groups(handle, of)
        ptrs, res, todo = self._outputs(handle, self._mean_parts(o, slots=True), slots=True, host="mean_slots")
        if todo:
            self._check(self._lib.magent_b200_get_mean_action_slots(self.game, g, o, *ptrs), "get_mean_action_slots")
        return res

    def get_mean_action_slots_torch(self, handle, of=None, out=None):
        """the slot-ordered mean neighbour action (see get_mean_action_slots) written straight into CUDA tensors, without
        waiting for the device: (mean float32 (num_arenas, S, n_action(of)), count int32 (num_arenas, S)).

        out: a caller-owned pair (mean, count) of contiguous CUDA tensors of those shapes and dtypes; needed to record
        the call into a CUDA graph (capture_graph), since the call then allocates nothing once a first call has run.
        count may be None: it is then not written, and None comes back in its place."""
        g, o = self._groups(handle, of)
        ptrs, res, todo = self._outputs(handle, self._mean_parts(o, slots=True), slots=True, out=out)
        if todo:
            self._check(self._lib.magent_b200_get_mean_action_slots(self.game, g, o, *ptrs), "get_mean_action_slots")
        return res

    def get_neighbours_slots(self, handle, k, of=None):
        """(idx int32 (num_arenas, S, k), rel int32 (num_arenas, S, k, 2), count int32 (num_arenas, S)): the nearest
        visible neighbours (see get_neighbours) in the stable slot layout (see get_slots).  idx holds each neighbour's
        flat slot a * S_of + slot in group `of` (S_of = get_slot_space(of)) instead of its row, so it stays valid for the
        episode: after clear_dead it may name a vacant slot, never another agent.  Unused entries and vacant slots are
        -1, with count 0.  The arrays are cached receive buffers: valid until the next call."""
        g, o = self._groups(handle, of)
        k, parts = self._nbr_parts(k)
        ptrs, res, todo = self._outputs(handle, parts, slots=True, host="nbr_slots")
        if todo:
            self._check(self._lib.magent_b200_get_neighbours_slots(self.game, g, o, k, *ptrs), "get_neighbours_slots")
        return res

    def get_neighbours_slots_torch(self, handle, k, of=None, out=None):
        """the slot-ordered nearest visible neighbours (see get_neighbours_slots) written straight into CUDA tensors,
        without waiting for the device: (idx int32 (num_arenas, S, k), rel int32 (num_arenas, S, k, 2), count int32
        (num_arenas, S)).  Gather slot-ordered features of group `of` with hid_s.view(-1, d)[idx.clamp(min=0)].

        out: a caller-owned triple (idx, rel, count) of contiguous CUDA int32 tensors of those shapes; needed to record
        the call into a CUDA graph (capture_graph), since the call then allocates nothing once a first call has run.  rel
        and count may be None: they are then neither computed nor written (without count the kernel stops at the k-th
        neighbour), and None comes back in their place."""
        g, o = self._groups(handle, of)
        k, parts = self._nbr_parts(k)
        ptrs, res, todo = self._outputs(handle, parts, slots=True, out=out)
        if todo:
            self._check(self._lib.magent_b200_get_neighbours_slots(self.game, g, o, k, *ptrs), "get_neighbours_slots")
        return res

    # ---- built-in scripted opponents (include/magent_b200_ext.h magent_b200_rule_actions has the definition)
    RULE_POLICIES = {"rush": 0, "flee": 1}

    def _rule_args(self, handle, target, policy, seed):
        if isinstance(policy, str):
            if policy not in self.RULE_POLICIES:
                raise ValueError("policy must be one of %s, got %r" % (sorted(self.RULE_POLICIES), policy))
            policy = self.RULE_POLICIES[policy]
        return self.game, self._hv(handle), self._hv(target), int(policy), int(seed)

    def set_rule_actions(self, handle, target, policy="rush", seed=0):
        """set_action with the built-in scripted opponent's choice for every agent of the group, decided on the device
        against group `target`: "rush" attacks the weakest target in reach, else steps towards the nearest visible one;
        "flee" steps away from the nearest visible one; both fall back to the draw of set_random_legal_actions(handle,
        seed).  Nothing waits for the device, and the call can be recorded into a CUDA graph (capture_graph)."""
        self._check(self._lib.magent_b200_rule_actions(*self._rule_args(handle, target, policy, seed)),
                    "rule_actions")

    def get_rule_actions(self, handle, target, policy="rush", seed=0):
        """int32 (n,): the actions set_rule_actions would set, in the order of set_action.  The array is a cached
        receive buffer: valid until the next call."""
        (ptr,), (act,), todo = self._outputs(handle, self._RULE_PARTS, host="rule")
        self._check(self._lib.magent_b200_get_rule_actions(*self._rule_args(handle, target, policy, seed),
                                                           ptr if todo else None), "get_rule_actions")
        return act

    def get_rule_actions_torch(self, handle, target, policy="rush", seed=0, out=None):
        """the scripted actions (see get_rule_actions) written straight into a CUDA int32 tensor (n,).

        out: a caller-owned contiguous CUDA int32 tensor (rows,) with at least get_num_bound(handle) rows; needed to
        record the call into a CUDA graph (capture_graph), since the call then allocates nothing.  Returns its first
        get_num(handle) entries."""
        (ptr,), (act,), todo = self._outputs(handle, self._RULE_PARTS, out=out)
        if todo:
            self._check(self._lib.magent_b200_get_rule_actions(*self._rule_args(handle, target, policy, seed), ptr),
                        "get_rule_actions")
        return act

    def get_rule_actions_slots(self, handle, target, policy="rush", seed=0):
        """int32 (num_arenas, S): the scripted actions (see get_rule_actions) in the stable slot layout (see get_slots);
        -1 in vacant slots.  The array is a cached receive buffer: valid until the next call."""
        (ptr,), (act,), todo = self._outputs(handle, self._RULE_PARTS, slots=True, host="rule_slots")
        self._check(self._lib.magent_b200_get_rule_actions_slots(*self._rule_args(handle, target, policy, seed),
                                                                 ptr if todo else None), "get_rule_actions_slots")
        return act

    def get_rule_actions_slots_torch(self, handle, target, policy="rush", seed=0, out=None):
        """the slot-ordered scripted actions (see get_rule_actions_slots) written straight into a CUDA int32 tensor
        (num_arenas, S), without waiting for the device.

        out: a caller-owned contiguous CUDA int32 tensor of that shape; needed to record the call into a CUDA graph
        (capture_graph), since the call then allocates nothing once a first call has run."""
        (ptr,), (act,), todo = self._outputs(handle, self._RULE_PARTS, slots=True, out=out)
        self._check(self._lib.magent_b200_get_rule_actions_slots(*self._rule_args(handle, target, policy, seed),
                                                                 ptr if todo else None), "get_rule_actions_slots")
        return act

    def get_counters(self):
        """int64 event counters accumulated on the device since construction"""
        buf = (ctypes.c_longlong * 16)()
        n = self._lib.magent_b200_get_counters(self.game, buf, 16)
        return [int(buf[i]) for i in range(n)]

    def sync(self):
        self._lib.magent_b200_sync(self.game)

    def get_io_stats(self):
        """step-loop traffic so far: dict(d2h=PCIe device->host bytes, h2d=..., host_written=bytes the engine's host
        threads wrote into caller buffers)"""
        buf = (ctypes.c_longlong * 6)()
        self._lib.magent_b200_get_io_stats(self.game, buf, 6)
        return {"d2h": int(buf[0]), "h2d": int(buf[1]), "host_written": int(buf[2]),
                "us_wire": int(buf[3]), "us_expand": int(buf[4]), "us_feature": int(buf[5])}

    def capture_graph(self, fn):
        """record the step-loop calls fn() makes (CUDA device pointers only, an even number of clear_dead) into a CUDA
        graph; returns its id for launch_graph"""
        self._lib.magent_b200_graph_begin(self.game)
        fn()
        return int(self._lib.magent_b200_graph_end(self.game))

    def launch_graph(self, graph_id, times=1):
        self._lib.magent_b200_graph_launch(self.game, int(graph_id), int(times))

    def step_device_done(self, done_ptr):
        """env_step with a CUDA device int for `done`: returns without waiting for the step (device-resident loops)"""
        self._lib.env_step(self.game, ctypes.cast(ctypes.c_void_p(int(done_ptr)), ctypes.POINTER(ctypes.c_int)))

    def set_profiling(self, on):
        """bracket every obs-render kernel launch with CUDA events (adds a sync per launch)"""
        self._lib.magent_b200_set_profiling(self.game, 1 if on else 0)

    def get_profile(self):
        """(total obs-render kernel milliseconds, launches) since profiling was enabled"""
        ms = ctypes.c_double(0.0)
        n = ctypes.c_longlong(0)
        self._lib.magent_b200_get_profile(self.game, ctypes.byref(ms), ctypes.byref(n))
        return ms.value, n.value

    def _set_obs_launch(self, grid=0, chunk=0, tile=0):
        """force the observation render's launch shape of this engine (tests): CTAs, consecutive tiles per CTA visit,
        tile width 1 narrow / 2 wide; 0 = automatic.  Raises ValueError (and changes nothing) on a refused value."""
        keys = (b"obs_grid", b"obs_chunk", b"obs_tile")
        old = self._get_obs_override()
        for key, value in zip(keys, (grid, chunk, tile)):
            if self._lib.env_config_game(self.game, key, _cint(int(value))) < 0:
                why = self._lib.magent_b200_last_error().decode()
                for k, v in zip(keys, old):
                    self._lib.env_config_game(self.game, k, _cint(v))
                raise ValueError(why)

    def _get_obs_override(self):
        """(grid, chunk, tile) as set by _set_obs_launch"""
        buf = np.zeros((3,), dtype=np.int32)
        self._lib.env_get_info(self.game, -1, b"obs_override", buf.ctypes.data)
        return tuple(int(v) for v in buf)

    def _get_obs_launch(self):
        """the last render launch of this engine: dict(elem_bytes, nit, turn, tile_agents, grid, chunk, tiles, aligned)"""
        buf = np.zeros((8,), dtype=np.int32)
        self._check(self._lib.env_get_info(self.game, -1, b"obs_launch", buf.ctypes.data), "obs_launch")
        keys = ("elem_bytes", "nit", "turn", "tile_agents", "grid", "chunk", "tiles", "aligned")
        return dict(zip(keys, (int(v) for v in buf)))

    def _get_step_launch(self):
        """the last step and cull launches of this engine: two dicts(mode (0 a CTA per arena, 1 the whole-grid team),
        grid, threads, smem, scratch_in_smem); all zero before the first launch"""
        buf = np.zeros((10,), dtype=np.int32)
        self._check(self._lib.env_get_info(self.game, -1, b"step_launch", buf.ctypes.data), "step_launch")
        keys = ("mode", "grid", "threads", "smem", "scratch_in_smem")
        return tuple(dict(zip(keys, (int(v) for v in buf[k:k + 5]))) for k in (0, 5))

    def launch_count(self):
        """number of kernels this library has launched in this process"""
        return int(self._lib.magent_b200_launch_count())

    # ------------------------------------------------------------------ reward DSL -> ABI
    def _serialize_event_exp(self, config):
        """Number symbols and event nodes and send them to the engine.

        The numbering must match the reference exactly (gridworld.py:493-565): symbol numbers fix
        the binding order of the rule evaluation (RewardEngine.cc:156-189 iterates a std::set of
        symbol pointers), so: per rule, receivers first, then a pre-order walk of the trigger.
        """
        L, game = self._lib, self.game
        sym_no, node_no = {}, {}

        def number_symbols(node):
            for item in node.inputs:
                if isinstance(item, EventNode):
                    number_symbols(item)
                elif isinstance(item, AgentSymbol) and item not in sym_no:
                    sym_no[item] = len(sym_no)

        def number_nodes(node):
            if node not in node_no:
                node_no[node] = len(node_no)
            for item in node.inputs:
                if isinstance(item, EventNode):
                    number_nodes(item)

        for on, receivers, _values, _terminal in config.reward_rules:
            for sym in receivers:
                if sym not in sym_no:
                    sym_no[sym] = len(sym_no)
            number_symbols(on)
        for rule in config.reward_rules:
            number_nodes(rule[0])
        config.symbol_ct, config.node_ct = len(sym_no), len(node_no)

        for sym, no in sym_no.items():
            L.gridworld_define_agent_symbol(game, no, sym.group, sym.index)

        for node, no in node_no.items():
            raw = np.zeros((len(node.inputs),), dtype=np.int32)
            for i, item in enumerate(node.inputs):
                if isinstance(item, EventNode):
                    raw[i] = node_no[item]
                elif isinstance(item, AgentSymbol):
                    raw[i] = sym_no[item]
                else:
                    raw[i] = item
            L.gridworld_define_event_node(game, no, node.op, as_int32_c_array(raw), len(raw))

        for on, receivers, values, terminal in config.reward_rules:
            recv = np.array([sym_no[s] for s in receivers], dtype=np.int32)
            auto = len(values) == 1 and values[0] == "auto"
            val = (np.zeros((len(recv),), dtype=np.float32) if auto
                   else np.array(values, dtype=np.float32))
            L.gridworld_add_reward_rule(game, node_no[on], as_int32_c_array(recv),
                                        as_float_c_array(val), len(recv), bool(terminal), bool(auto))


# ---------------------------------------------------------------------- reward description DSL
class EventNode:
    """AST node of an event expression (reference: gridworld.py:571-650).

    Leaves are built by calling the module-level ``Event`` object:
    ``Event(subject, 'attack', target)``; nodes combine with ``&``, ``|`` and ``~``.
    Operator numbers follow src/gridworld/grid_def.h:17-23.
    """
    OP_AND, OP_OR, OP_NOT = 0, 1, 2
    OP_KILL, OP_AT, OP_IN, OP_COLLIDE, OP_ATTACK, OP_DIE = 3, 4, 5, 6, 7, 8
    OP_IN_A_LINE, OP_ALIGN = 9, 10

    _BINARY_AGENT = {"kill": OP_KILL, "attack": OP_ATTACK, "collide": OP_COLLIDE}
    _UNARY_AGENT = {"die": OP_DIE, "in_a_line": OP_IN_A_LINE, "align": OP_ALIGN}

    def __init__(self, op=None, inputs=(), predicate=None):
        self.op = op
        self.predicate = predicate
        self.inputs = list(inputs)

    def __call__(self, subject, predicate, *args):
        if predicate in self._BINARY_AGENT:
            return EventNode(self._BINARY_AGENT[predicate], [subject, args[0]], predicate)
        if predicate in self._UNARY_AGENT:
            return EventNode(self._UNARY_AGENT[predicate], [subject], predicate)
        if predicate == "at":
            x, y = args[0][0], args[0][1]
            return EventNode(self.OP_AT, [subject, x, y], predicate)
        if predicate == "in":
            (ax, ay), (bx, by) = args[0][0], args[0][1]
            return EventNode(self.OP_IN,
                             [subject, min(ax, bx), min(ay, by), max(ax, bx), max(ay, by)], predicate)
        raise Exception("invalid predicate of event " + predicate)

    def __and__(self, other):
        return EventNode(self.OP_AND, [self, other])

    def __or__(self, other):
        return EventNode(self.OP_OR, [self, other])

    def __invert__(self):
        return EventNode(self.OP_NOT, [self])


Event = EventNode()


class AgentSymbol:
    """symbol standing for some agent(s) of a group (reference: gridworld.py:654-675)

    index: 'any' (-1), 'all' (-2) or a deterministic int index into the group.
    """

    def __init__(self, group, index):
        self.group = group if group is not None else -1
        if index == "any":
            self.index = -1
        elif index == "all":
            self.index = -2
        else:
            assert isinstance(index, (int, np.integer)), "index must be a deterministic int"
            self.index = int(index)

    def __str__(self):
        return "agent(%d,%d)" % (self.group, self.index)


class Config:
    """game configuration (reference: gridworld.py:678-766)"""

    def __init__(self):
        self.config_dict = {}
        self.agent_type_dict = {}
        self.groups = []
        self.reward_rules = []

    def set(self, args):
        """global key/value pairs, e.g. {"map_width": 100, "minimap_mode": True}"""
        self.config_dict.update(args)

    def register_agent_type(self, name, attr):
        """register an agent type; attr keys as in src/gridworld/AgentType.cc:52-78
        (width, length, speed, hp, view_range, attack_range, damage, step_recover, kill_supply,
        step_reward, kill_reward, dead_penalty, attack_penalty, attack_in_group, ...)"""
        if name in self.agent_type_dict:
            raise Exception("type name %s already exists" % name)
        self.agent_type_dict[name] = attr
        return name

    def add_group(self, agent_type):
        """returns the handle (an int) of the new group"""
        self.groups.append(agent_type)
        return len(self.groups) - 1

    def add_reward_rule(self, on, receiver, value, terminal=False):
        """when event ``on`` holds, give ``value`` to ``receiver`` (lists allowed)"""
        if not isinstance(receiver, (tuple, list)):
            assert not isinstance(value, (tuple, list))
            receiver, value = [receiver], [value]
        if len(receiver) != len(value):
            raise Exception("the length of receiver and value should be equal")
        self.reward_rules.append([on, list(receiver), list(value), terminal])


class CircleRange:
    """circular view/attack range (reference: gridworld.py:769-781)"""

    def __init__(self, radius):
        self.radius = radius
        self.angle = 360

    def __str__(self):
        return "circle(%g)" % self.radius


class SectorRange:
    """sector view/attack range, angle < 180 (reference: gridworld.py:784-800)"""

    def __init__(self, radius, angle):
        self.radius = radius
        self.angle = angle
        if self.angle >= 180:
            raise Exception("the angle of a sector should be smaller than 180 degree")

    def __str__(self):
        return "sector(%g, %g)" % (self.radius, self.angle)
