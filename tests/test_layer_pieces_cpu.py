"""The SASRec, TIGER and COBRA layers share one definition of each piece whose copies could drift without failing: the
feed-forward pair (genrec_b200.functional.ffn_fwd / ffn_bwd, whose backward must re-derive the dropout masks of its forward),
the dropout seed rule (dropout_seed, StepSeeds._seeds) and the zero-bias cache.  A layer that calls the FFN's epilogue GEMMs
itself, reads torch.initial_seed itself or keeps its own cache or step counter is a second copy."""
import ast
import glob
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FFN_GEMMS = ("linear_dact_bwd", "linear_residual_fwd")


def _trees():
    paths = sorted(glob.glob(os.path.join(ROOT, "genrec_b200", "*.py")))
    return {os.path.basename(p): ast.parse(open(p).read(), p) for p in paths}


def _called(node):
    f = node.func
    return f.attr if isinstance(f, ast.Attribute) else f.id if isinstance(f, ast.Name) else None


def _copies(tree):
    for node in ast.walk(tree):
        if isinstance(node, ast.Call) and _called(node) in FFN_GEMMS:
            yield node.lineno, f"calls {_called(node)}"
        elif isinstance(node, ast.Attribute) and node.attr == "initial_seed":
            yield node.lineno, "reads torch.initial_seed"


def _zero_bias_cache(node):
    return (isinstance(node, ast.FunctionDef) and node.name.lstrip("_") == "zero_bias") or \
        (isinstance(node, ast.Name) and "ZERO_BIAS" in node.id)


def _step_counter(node):
    return isinstance(node, ast.FunctionDef) and node.name == "_seeds"


def _definitions(trees, is_def):
    return [(name, node.lineno) for name, tree in trees.items() for node in ast.walk(tree) if is_def(node)]


def test_layers_build_on_the_shared_pieces():
    trees = _trees()
    assert {"functional.py", "sasrec.py", "tiger.py", "cobra.py", "t5_attention.py", "hstu.py"} <= set(trees)
    bad = {name: list(_copies(tree)) for name, tree in trees.items() if name != "functional.py"}
    assert not {k: v for k, v in bad.items() if v}
    # the pieces are there, in functional.py: the check above is not passing on an empty tree
    calls = {_called(n) for n in ast.walk(trees["functional.py"]) if isinstance(n, ast.Call)}
    assert set(FFN_GEMMS) <= calls
    defs = {n.name for n in ast.walk(trees["functional.py"]) if isinstance(n, (ast.FunctionDef, ast.ClassDef))}
    assert {"ffn_fwd", "ffn_bwd", "matmul_f32", "dropout_seed", "zero_bias", "StepSeeds", "_seeds"} <= defs


def test_one_zero_bias_cache_and_one_step_counter():
    trees = _trees()
    assert [f for f, _ in _definitions(trees, _zero_bias_cache)] == ["functional.py"]
    assert [f for f, _ in _definitions(trees, _step_counter)] == ["functional.py"]
