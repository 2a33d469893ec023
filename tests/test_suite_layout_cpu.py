"""Test modules import support modules (tests/*.py not named test_*) and never another test module, so that renaming a helper
breaks only the modules that name it, and the CPU tests need no GPU test module."""
import ast
import glob
import os


def _test_module_imports(path):
    for node in ast.walk(ast.parse(open(path).read(), path)):
        if isinstance(node, ast.Import):
            yield from (a.name for a in node.names if a.name.startswith("tests.test_"))
        elif isinstance(node, ast.ImportFrom) and node.module:
            if node.module.startswith("tests.test_"):
                yield node.module
            elif node.module == "tests":
                yield from ("tests." + a.name for a in node.names if a.name.startswith("test_"))


def test_no_test_module_imports_another():
    here = os.path.dirname(os.path.abspath(__file__))
    paths = sorted(glob.glob(os.path.join(here, "test_*.py")))
    assert os.path.abspath(__file__) in paths
    bad = {os.path.basename(p): sorted(set(_test_module_imports(p))) for p in paths}
    assert not {k: v for k, v in bad.items() if v}
