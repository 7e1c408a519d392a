"""The reference's own kernels (oracle/_ref/libjvector.so) as the tests call them, live or replayed from a recording.

Where the reference library has been built, the `ref` fixture calls it directly; with JV_RECORD_REF=1 it also records every
call (name, scalar arguments, return value, bytes written to the output buffer) under tests/golden/ref/<test module>.npz.
Everywhere else the fixture replays that recording in call order: the tests compute the same seeded inputs, so the reference's
answers come back for exactly the inputs they were recorded on, and a call whose name or scalar arguments differ from the
recording fails the test."""
import ctypes as C
import json
import os

import numpy as np

import oracle_lib as o

GOLDEN_DIR = os.path.join(o.GOLDEN, "ref")

# functions that write through a pointer: name -> (argument index, dtype, first element, element count), from the reference ABI
OUTPUTS = {
    "add_in_place_f32": (0, np.float32, lambda a: 0, lambda a: a[2]),
    "sub_in_place_f32": (0, np.float32, lambda a: 0, lambda a: a[2]),
    "min_in_place_f32": (0, np.float32, lambda a: 0, lambda a: a[2]),
    "add_scalar_in_place_f32": (0, np.float32, lambda a: 0, lambda a: a[2]),
    "sub_scalar_in_place_f32": (0, np.float32, lambda a: 0, lambda a: a[2]),
    "nvq_shuffle_query_in_place_8bit": (0, np.float32, lambda a: 0, lambda a: a[1]),
    "nvq_quantize_8bit": (6, np.uint8, lambda a: 0, lambda a: a[1]),
    "calculate_partial_sums_dot_f32": (6, np.float32, lambda a: a[1] * a[3], lambda a: a[3]),
    "calculate_partial_sums_euclidean_f32": (6, np.float32, lambda a: a[1] * a[3], lambda a: a[3]),
    "calculate_partial_sums_self_magnitude_f32": (4, np.float32, lambda a: a[1] * a[3], lambda a: a[3]),
}


def _view(ptr, dtype, first, count):
    ct = np.ctypeslib.as_ctypes_type(np.dtype(dtype))
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ct)), shape=(first + count,))[first:]


def _scalars(args):
    return [x if isinstance(x, (int, float)) and not isinstance(x, bool) else None for x in args]


def _path(module):
    return os.path.join(GOLDEN_DIR, module.replace(".py", "") + ".npz")


class Live:
    """The built reference library; `log` (a list) receives the calls when recording."""

    def __init__(self, lib, log=None):
        self._lib, self._log = lib, log

    def _record(self, name, scalars, ret, out):
        if self._log is not None:
            self._log.append(([name, scalars, ret], out))

    def __getattr__(self, name):
        if name.startswith("_"):
            raise AttributeError(name)
        fn = getattr(self._lib, name)

        def call(*args):
            ret = fn(*args)
            out = b""
            if name in OUTPUTS:
                i, dt, first, count = OUTPUTS[name]
                out = _view(args[i], dt, first(args), count(args)).tobytes()
            self._record(name, _scalars(args), ret, out)
            return ret
        return call

    def capture(self, label, fn):
        """fn() computes something from the reference library (a numpy array or a JSON value); recorded like a call"""
        value = fn()
        if isinstance(value, np.ndarray):
            self._record(label, [], {"dtype": value.dtype.str, "shape": list(value.shape)}, value.tobytes())
        else:
            self._record(label, [], value, b"")
        return value


class Replay:
    def __init__(self, test, calls, out):
        self._test, self._calls, self._out, self._i, self._pos = test, calls, out, 0, 0

    def _next(self, name, scalars):
        if self._i >= len(self._calls):
            raise AssertionError("%s: more reference calls than recorded (call %d: %s)" % (self._test, self._i, name))
        (rname, rscalars, ret), nbytes = self._calls[self._i]
        if rname != name or rscalars != scalars:
            raise AssertionError("%s: reference call %d recorded as %s%s, called as %s%s" % (self._test, self._i, rname, rscalars, name, scalars))
        self._i += 1
        blob = self._out[self._pos:self._pos + nbytes]
        self._pos += nbytes
        return ret, blob

    def __getattr__(self, name):
        if name.startswith("_"):
            raise AttributeError(name)

        def call(*args):
            ret, blob = self._next(name, _scalars(args))
            if name in OUTPUTS:
                i, dt, first, count = OUTPUTS[name]
                _view(args[i], dt, first(args), count(args))[:] = np.frombuffer(blob, dt)
            return ret
        return call

    def capture(self, label, fn):
        ret, blob = self._next(label, [])
        if isinstance(ret, dict) and "dtype" in ret:
            return np.frombuffer(blob, np.dtype(ret["dtype"])).reshape(ret["shape"]).copy()
        return ret


class Session:
    """One per pytest session: hands each test its `ref` and writes the recording at the end."""

    def __init__(self):
        self.lib = o.load_ref()
        self.record = self.lib is not None and os.environ.get("JV_RECORD_REF") == "1"
        self.logs = {}  # module -> {test: [(call, bytes)]}
        self.cache = {}

    def for_test(self, module, test):
        if self.lib is not None:
            log = None
            if self.record:
                log = self.logs.setdefault(module, {}).setdefault(test, [])
                del log[:]
            return Live(self.lib, log)
        if module not in self.cache:
            p = _path(module)
            self.cache[module] = None
            if os.path.exists(p):
                z = np.load(p)
                self.cache[module] = (json.loads(bytes(z["index"]).decode()), z["out"].tobytes())
        rec = self.cache[module]
        if rec is None or test not in rec[0]:
            return None
        calls, start = rec[0][test]
        nbytes = sum(n for _, n in calls)
        return Replay(test, calls, rec[1][start:start + nbytes])

    def close(self):
        for module, tests in self.logs.items():
            p = _path(module)
            index, blobs, pos = {}, [], 0
            if os.path.exists(p):  # keep the tests of this module that this session did not run
                z = np.load(p)
                old_index, old_out = json.loads(bytes(z["index"]).decode()), z["out"].tobytes()
                for t, (calls, start) in old_index.items():
                    if t not in tests:
                        n = sum(c[1] for c in calls)
                        index[t] = (calls, pos)
                        blobs.append(old_out[start:start + n])
                        pos += n
            for t, log in sorted(tests.items()):
                index[t] = ([(c, len(b)) for c, b in log], pos)
                for _, b in log:
                    blobs.append(b)
                    pos += len(b)
            os.makedirs(GOLDEN_DIR, exist_ok=True)
            np.savez_compressed(p, index=np.frombuffer(json.dumps(index).encode(), np.uint8),
                                out=np.frombuffer(b"".join(blobs), np.uint8))
