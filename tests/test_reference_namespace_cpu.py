"""Every Python module of the reference package imports under the same dotted name here (``ppfleetx.<path>``), and the public names it
defines at module level exist in ours.  This is the "switch the import and keep going" contract of the ``ppfleetx`` alias package."""
import ast
import importlib
import json
import os

import golden_ref

GOLDEN = os.path.join(golden_ref.GOLDEN_DIR, "reference_namespace.json")      # {module name below ppfleetx: "public names"}
_SKIP_PREFIX = ("_",)


def _public_defs(path):
    tree = ast.parse(open(path, encoding="utf-8").read())
    out = []
    for node in tree.body:
        if isinstance(node, (ast.ClassDef, ast.FunctionDef)) and not node.name.startswith(_SKIP_PREFIX):
            out.append(node.name)
    return out


def _reference_modules():
    """(module name, public names) of every module of the original package: from the stored list, or from a checkout (which rewrites the list)."""
    if not golden_ref.REFERENCE_DIR:
        with open(GOLDEN, encoding="utf-8") as f:
            return sorted((("ppfleetx." + k).rstrip("."), v.split()) for k, v in json.load(f).items())
    ref, found = os.path.join(golden_ref.REFERENCE_DIR, "ppfleetx"), {}
    for dirpath, _, files in os.walk(ref):
        for f in sorted(files):
            if f.endswith(".py"):
                rel = os.path.relpath(os.path.join(dirpath, f), os.path.dirname(ref))[:-3]
                name = rel.replace(os.sep, ".")
                found[name[:-len(".__init__")] if name.endswith(".__init__") else name] = _public_defs(os.path.join(dirpath, f))
    with open(GOLDEN, "w", encoding="utf-8") as f:
        json.dump({k[len("ppfleetx"):].lstrip("."): " ".join(v) for k, v in found.items()}, f, separators=(",", ":"), sort_keys=True)
        f.write("\n")
    return sorted(found.items())


def test_every_reference_module_name_imports():
    missing = []
    n = 0
    for name, _ in _reference_modules():
        n += 1
        try:
            importlib.import_module(name)
        except Exception as e:          # noqa: BLE001 - the report wants every failure, whatever its type
            missing.append(f"{name}: {type(e).__name__}: {e}")
    assert n > 150
    assert not missing, "\n".join(missing)


# public names of the reference not provided yet, one ``module.name`` per line; the test fails when a name outside this file goes missing AND
# when a listed name has been provided (so the file can only shrink)
_KNOWN_GAPS_FILE = os.path.join(os.path.dirname(__file__), "reference_namespace_known_gaps.txt")


def _known_gaps():
    if not os.path.exists(_KNOWN_GAPS_FILE):
        return set()
    with open(_KNOWN_GAPS_FILE, encoding="utf-8") as f:
        return {line.strip() for line in f if line.strip() and not line.startswith("#")}


def test_public_classes_and_functions_exist():
    absent = set()
    total = 0
    for name, defs in _reference_modules():
        try:
            mod = importlib.import_module(name)
        except Exception:               # noqa: BLE001 - reported by the test above
            continue
        for sym in defs:
            total += 1
            if not hasattr(mod, sym):
                absent.add(f"{name}.{sym}")
    assert total > 500
    known = _known_gaps()
    new_gaps, closed = sorted(absent - known), sorted(known - absent)
    assert not new_gaps, f"{len(new_gaps)} of {total} public names missing:\n" + "\n".join(new_gaps)
    assert not closed, "provided now, remove from reference_namespace_known_gaps.txt:\n" + "\n".join(closed)
