"""The reference's own code as the tests see it: recorded answers of ref_api (oracle/_ref/libvxref.so, the reference's sources compiled
against oracle/ref_standin) replayed in call order, so that a test comparing the oracle with the reference runs in any checkout.

reference() stands in for the ref_api module.  Every call made through it (module functions, constructors, methods of the objects they return)
yields the value the reference returned when the tape was recorded.  Tapes live in tests/golden/ref_pin/<test>.npz: the call results as a JSON
tree plus the arrays they contain, bit for bit.  Every array is stored whole as long as the tape file stays within FILE_BUDGET; only a tape that
would not fit has its largest numeric arrays cut, largest first and each by half at a time, to a fixed, seeded sample of rows (axis 0; the sample
of a shorter cut is part of a longer one, so arrays of one length share rows).  A cut array comes back as a masked array whose other rows are
masked, so the comparisons of a test see exactly the recorded rows.  The fields the tests sort or match voxels by (WHOLE) are never cut.

Recording needs the reference build (oracle/_ref/libvxref.so):   VXS_RECORD_REFERENCE=1 python -m pytest tests/test_ref_pin.py
The inputs are not stored: the tests re-create them from their seeded generators."""
import json
import os

import numpy as np

TAPES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_pin")
RECORD = os.environ.get("VXS_RECORD_REFERENCE") == "1"
FILE_BUDGET = 960_000          # bytes per tape file
WHOLE = ("sum10", "voxel_center")


class _Tape:
    def __init__(self):
        self.name, self.items, self.arrays, self.cuttable, self.pos = None, [], {}, set(), 0

    def begin(self, name):
        self.name, self.items, self.arrays, self.cuttable, self.pos = name, [], {}, set(), 0
        if not RECORD:
            z = np.load(os.path.join(TAPES, name + ".npz"))
            tape = json.loads(str(z["tape"]))
            blob = z["blob"].tobytes()
            self.items = tape["items"]
            for k, (dt, shape, off, rows) in tape["arrays"].items():
                dt = np.dtype([tuple(f) for f in dt] if isinstance(dt, list) else dt)
                n = int(np.prod(shape, dtype=np.int64)) * dt.itemsize
                a = np.frombuffer(blob[off:off + n], dtype=dt).reshape(shape)
                if rows is not None:                # a cut array: rows = its full length; the kept rows are the seeded prefix
                    keep = _rows(rows, shape[0])
                    full = np.zeros((rows,) + tuple(shape[1:]), dtype=dt)
                    full[keep] = a
                    mask = np.ones(full.shape, dtype=bool)
                    mask[keep] = False
                    a = np.ma.masked_array(full, mask)
                self.arrays[k] = a

    def _save(self, keep):
        """Writes the tape with array k cut to its first keep[k] sampled rows; returns the file size."""
        meta, parts, off = {}, [], 0          # every array of the tape in one byte blob: a tape holds hundreds of small arrays
        for k, a in self.arrays.items():
            full = a.shape[0] if k in keep else None
            a = np.ascontiguousarray(a[_rows(a.shape[0], keep[k])] if k in keep else a)
            meta[k] = [a.dtype.descr if a.dtype.names else a.dtype.str, list(a.shape), off, full]
            parts.append(a.tobytes()); off += a.nbytes
        path = os.path.join(TAPES, self.name + ".npz")
        np.savez_compressed(path, tape=np.array(json.dumps({"items": self.items, "arrays": meta})), blob=np.frombuffer(b"".join(parts), dtype=np.uint8))
        return os.path.getsize(path)

    def end(self):
        if RECORD and self.name is not None:
            os.makedirs(TAPES, exist_ok=True)
            keep = {}
            while self._save(keep) > FILE_BUDGET:
                rowbytes = {k: self.arrays[k].nbytes // self.arrays[k].shape[0] for k in self.cuttable}
                k = max((k for k in self.cuttable if keep.get(k, self.arrays[k].shape[0]) > 1), key=lambda k: keep.get(k, self.arrays[k].shape[0]) * rowbytes[k])
                keep[k] = keep.get(k, self.arrays[k].shape[0]) // 2
        elif self.name is not None:
            assert self.pos == len(self.items), f"{self.name}: {len(self.items) - self.pos} recorded reference calls were not replayed"
        self.name = None

    def put(self, v, field=None):
        """Encodes a call result (data only: the objects a call returns are handled by call())."""
        if v is None or isinstance(v, (bool, int, float, str)):
            return v
        if isinstance(v, (np.generic,)) and v.dtype.kind in "biuf":
            return {"s": v.dtype.str, "v": v.item()}
        if isinstance(v, np.ndarray):
            k = f"a{len(self.arrays)}"
            self.arrays[k] = v.copy()
            if v.dtype.kind in "biuf" and v.ndim > 0 and v.shape[0] > 1 and field not in WHOLE:
                self.cuttable.add(k)
            return {"a": k}
        if isinstance(v, (tuple, list)):
            return {"t" if isinstance(v, tuple) else "l": [self.put(x) for x in v]}
        if isinstance(v, dict):
            return {"d": {k: self.put(x, k) for k, x in v.items()}}
        raise TypeError(f"cannot record a {type(v).__name__} inside a call result")

    def get(self, e):
        if e is None or isinstance(e, (bool, int, float, str)):
            return e
        if "s" in e:
            return np.dtype(e["s"]).type(e["v"])
        if "a" in e:
            return self.arrays[e["a"]]
        if "t" in e:
            return tuple(self.get(x) for x in e["t"])
        if "l" in e:
            return [self.get(x) for x in e["l"]]
        if "d" in e:
            return {k: self.get(x) for k, x in e["d"].items()}
        return _Proxy(self, None)                     # {"o": 1}: an object of the reference build (factor, map, IMU window ...)

    def call(self, fn, args, kwargs):
        if RECORD:
            res = fn(*[_unwrap(a) for a in args], **{k: _unwrap(v) for k, v in kwargs.items()})
            is_data = res is None or isinstance(res, (bool, int, float, str, np.generic, np.ndarray, tuple, list, dict))
            self.items.append(self.put(res) if is_data else {"o": 1})
            return res if is_data else _Proxy(self, res)
        assert self.pos < len(self.items), f"{self.name}: more reference calls than were recorded"
        self.pos += 1
        return self.get(self.items[self.pos - 1])


def _rows(n, keep):
    """The first `keep` rows of the fixed permutation of n rows, in ascending order."""
    return np.sort(np.random.default_rng(n).permutation(n)[:keep])


def _unwrap(a):
    return a._real if isinstance(a, _Proxy) else a


class _Proxy:
    """A name reached through `ref` (module attribute, class, method, returned object)."""

    def __init__(self, tape, real):
        self._tape, self._real = tape, real

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return _Proxy(self._tape, getattr(self._real, name) if RECORD else None)

    def __call__(self, *args, **kwargs):
        return self._tape.call(self._real, args, kwargs)


tape = _Tape()


def reference():
    """The stand-in for the ref_api module (the real module when recording)."""
    real = None
    if RECORD:
        import ref_api
        assert ref_api.available(), "recording needs oracle/_ref/libvxref.so (built by oracle/Makefile where the reference sources exist)"
        real = ref_api
    return _Proxy(tape, real)
