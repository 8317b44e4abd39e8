"""Stand-ins for models built by the original project's constructors: what a parity test reads from such a model (tensor shapes, names) is
stored under ``tests/golden/<name>.json``, one record per constructor call, and replayed as meta tensors.  With ``PFX_REFERENCE_DIR`` set
to a checkout of the original project, every constructor call runs the original source and rewrites its record."""
import contextlib
import json
import os

import torch

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
REFERENCE_DIR = os.environ.get("PFX_REFERENCE_DIR", "")


def _key(x):
    if isinstance(x, _Model):
        return x.key
    if isinstance(x, dict):
        return "{" + ",".join(f"{k}={_key(v)}" for k, v in sorted(x.items())) + "}"
    if isinstance(x, (list, tuple)):
        return "(" + ",".join(_key(v) for v in x) + ")"
    return repr(x)


def _pack_names(names):
    """{pattern: [layer indices]}: the first integer component of a dotted name becomes ``#`` (``{pattern: []}`` for names without one)."""
    packed = {}
    for n in names:
        parts = n.split(".")
        i = next((j for j, x in enumerate(parts) if x.isdigit()), None)
        if i is None:
            packed.setdefault(n, [])
        else:
            packed.setdefault(".".join(parts[:i] + ["#"] + parts[i + 1:]), []).append(int(parts[i]))
    return packed


def _unpack_names(packed):
    return [pat.replace("#", str(i), 1) for pat, idx in packed.items() for i in idx] + [pat for pat, idx in packed.items() if not idx]


def _describe(model, names):
    seen, shapes = set(), {}
    for p in model.parameters():                   # distinct tensors, as torch reports them
        if id(p) not in seen:
            seen.add(id(p))
            shapes[tuple(p.shape)] = shapes.get(tuple(p.shape), 0) + 1
    rec = {"shapes": {"x".join(map(str, k)): n for k, n in shapes.items()}}        # "64x3x3x3": count ("" = a scalar)
    if names:
        rec["names"] = _pack_names(n for n, _ in model.named_parameters(remove_duplicate=False))
    if hasattr(model, "blocks"):
        rec["n_blocks"] = len(model.blocks)
    return rec


class _Model:
    """The parameters of a recorded model on the meta device: every distinct tensor once (``parameters()``), the tensor names (every name a tensor is
    reachable by) where the test asked for them (``named_parameters(remove_duplicate=False)``), the number of ``blocks``."""

    def __init__(self, key, rec, real=None):
        self.key, self.real, self._rec = key, real, rec
        self._params = [torch.empty(*[int(d) for d in shape.split("x") if d], device="meta") for shape, n in rec["shapes"].items() for _ in range(n)]
        if "n_blocks" in rec:
            self.blocks = range(rec["n_blocks"])

    def parameters(self):
        return iter(self._params)

    def named_parameters(self, remove_duplicate=True):
        assert not remove_duplicate, "only the names are stored, every alias included"
        return ((n, None) for n in _unpack_names(self._rec["names"]))


class _Namespace:
    """``ns.Ctor(...)`` / ``ns["Ctor"](...)`` of an original module: replayed from the store, or run and recorded when ``real`` is given."""

    def __init__(self, store, real=None, prefix="", names=False):
        self._store, self._real, self._prefix, self._names = store, real, prefix, names

    def __getattr__(self, name):
        if name.startswith("_"):
            raise AttributeError(name)
        return lambda *a, **kw: self._call(name, a, kw)

    __getitem__ = __getattr__

    def _call(self, name, a, kw):
        key = f"{self._prefix}{name}{_key(a)}{_key(kw)}"
        real = None
        if self._real is not None:
            ctor = self._real[name] if isinstance(self._real, dict) else getattr(self._real, name)
            real = ctor(*[x.real if isinstance(x, _Model) else x for x in a], **kw)
            self._store[key] = _describe(real, self._names)
        return _Model(key, self._store[key], real)


@contextlib.contextmanager
def namespaces(name, load_reference, count=1, names=False):
    """Yield ``count`` namespaces for the golden file ``name``.  ``load_reference`` is a context manager that yields the original module(s);
    it is entered only when recording.  ``names``: also store the parameter names."""
    path = os.path.join(GOLDEN_DIR, name + ".json")
    if not REFERENCE_DIR:
        with open(path, encoding="utf-8") as f:
            store = json.load(f)
        yield [_Namespace(store, prefix=f"{i}:") for i in range(count)]
        return
    store = {}
    with load_reference() as real:
        reals = list(real) if count > 1 else [real]
        yield [_Namespace(store, r, prefix=f"{i}:", names=names) for i, r in enumerate(reals)]
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    with open(path, "w", encoding="utf-8") as f:
        json.dump(store, f, separators=(",", ":"), sort_keys=True)
        f.write("\n")
