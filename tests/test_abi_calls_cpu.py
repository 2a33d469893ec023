"""The package reaches the C library only through genrec_b200/_lib.py: every other module launches with ``_lib.call`` and sizes
its scratch with ``_lib.workspace`` / ``_lib.host_bytes``, which pin each call to its device and that device's stream.  A module
that loads the library or names a ``grb_*`` symbol itself could skip the device guard or lose the library's error message."""
import ast
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _violations(path, entry_points):
    for node in ast.walk(ast.parse(open(path).read(), path)):
        if isinstance(node, ast.Call):
            f = node.func
            if (isinstance(f, ast.Attribute) and f.attr == "load" and isinstance(f.value, ast.Name) and f.value.id == "_lib") or \
                    (isinstance(f, ast.Name) and f.id == "load"):
                yield node.lineno, "_lib.load()"
        elif isinstance(node, ast.Attribute) and node.attr.startswith("grb_"):
            yield node.lineno, f"attribute {node.attr}"
        elif isinstance(node, ast.Constant) and isinstance(node.value, str) and re.fullmatch(r"grb_\w+", node.value):
            if node.value not in entry_points:
                yield node.lineno, f"{node.value!r} is not an entry point"


def _entry_point_literals(path):
    return [n.value for n in ast.walk(ast.parse(open(path).read(), path))
            if isinstance(n, ast.Constant) and isinstance(n.value, str) and re.fullmatch(r"grb_\w+", n.value)]


def test_only_the_stub_touches_the_library():
    from genrec_b200 import _lib
    paths = sorted(p for p in glob.glob(os.path.join(ROOT, "genrec_b200", "*.py")) if os.path.basename(p) != "_lib.py")
    assert os.path.join(ROOT, "genrec_b200", "functional.py") in paths
    bad = {os.path.basename(p): list(_violations(p, _lib.SIGNATURES)) for p in paths}
    assert not {k: v for k, v in bad.items() if v}
    # the calls are there, by name: the check above is not passing on an empty tree
    named = {n for p in paths for n in _entry_point_literals(p)}
    assert {"grb_hstu_layer_forward", "grb_linear_backward_workspace_bytes", "grb_sasrec_attention_forward"} <= named
