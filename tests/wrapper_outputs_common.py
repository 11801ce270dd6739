"""A recording proxy for the engine library, to hold the wrapper's calls to literal expectations."""
import ctypes

PTR, NULL = "ptr", "NULL"


def _null(a):
    v = a.value if isinstance(a, ctypes.c_void_p) else a
    return NULL if v is None or (isinstance(v, int) and v == 0) else PTR


def _arg(argtype, a):
    if argtype in (ctypes.c_int, ctypes.c_ulonglong):
        return int(a)
    if argtype is ctypes.c_char_p:
        return a.decode()
    if isinstance(a, ctypes.Array):
        return tuple(_null(x) for x in a)
    return _null(a)


class Recorder:
    """forwards every call to the engine library and logs it as (name, arguments after the engine handle): integers and
    info names as they are, pointers as PTR or NULL (an array of pointers as a tuple of those).  The host allocator's
    calls are not logged: how the wrapper caches its receive buffers is its own affair."""

    def __init__(self, lib):
        self._lib = lib
        self.log = []

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        argtypes = getattr(fn, "argtypes", None)
        if argtypes is None or name.startswith("magent_b200_host_"):
            return fn

        def call(*args):
            self.log.append((name,) + tuple(_arg(t, a) for t, a in zip(argtypes[1:], args[1:])))
            return fn(*args)
        return call

    def take(self):
        """the calls logged since the last take"""
        log, self.log = self.log, []
        return log


def num(g):
    return ("env_get_info", g, "num", PTR)


SLOT_SPACE = ("env_get_info", -1, "slot_space", PTR)
NUM_BOUND = ("env_get_info", -1, "num_bound", PTR)
