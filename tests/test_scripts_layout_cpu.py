"""The benchmark scripts measure through scripts/harness.py: one definition of how to describe the card, time a call eagerly or
from a CUDA graph, take peak memory, profile kernels and draw seeded workload lengths.  A script that keeps its own copy of one
of these, or imports another runnable script, is a copy that can drift from the others without failing."""
import ast
import glob
import os

import pytest
import torch

from scripts import harness

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HELPERS = {"card", "timed", "time_graph", "graphed", "kernel_us", "profile", "stage_of", "lengths_of", "peak", "graph_timed"}


def _trees():
    paths = sorted(glob.glob(os.path.join(ROOT, "scripts", "*.py")))
    return {os.path.basename(p): ast.parse(open(p).read(), p) for p in paths}


def _dotted(node):
    parts = []
    while isinstance(node, ast.Attribute):
        parts.append(node.attr)
        node = node.value
    if isinstance(node, ast.Name):
        parts.append(node.id)
    return ".".join(reversed(parts))


def _copies(tree):
    """(line, what) of every piece of the harness a script does itself"""
    for node in ast.walk(tree):
        if isinstance(node, (ast.FunctionDef, ast.AsyncFunctionDef)) and node.name in HELPERS:
            yield node.lineno, f"defines {node.name}"
        elif isinstance(node, ast.Call):
            name = _dotted(node.func)
            if name.endswith("CUDAGraph"):
                yield node.lineno, "constructs a CUDA graph"
            elif name.endswith("Event") and any(k.arg == "enable_timing" for k in node.keywords):
                yield node.lineno, "constructs a timing event"
            elif name.endswith("profiler.profile"):
                yield node.lineno, "constructs torch.profiler.profile"
        elif isinstance(node, ast.ImportFrom) and node.module == "torch.profiler" and any(a.name == "profile" for a in node.names):
            yield node.lineno, "imports torch.profiler.profile"
        elif isinstance(node, ast.Constant) and isinstance(node.value, str) and "nvidia-smi" in node.value:
            yield node.lineno, "names nvidia-smi"
        elif isinstance(node, ast.Import):
            yield from ((node.lineno, f"imports {a.name}") for a in node.names
                        if a.name.startswith("scripts.") and a.name != "scripts.harness")
        elif isinstance(node, ast.ImportFrom) and node.module and node.module.split(".")[0] == "scripts":
            names = [node.module + "." + a.name for a in node.names] if node.module == "scripts" else [node.module]
            yield from ((node.lineno, f"imports {n}") for n in names if n != "scripts.harness")


def test_scripts_measure_through_the_harness():
    trees = _trees()
    assert {"harness.py", "bench_kernels.py", "bench_cobra.py", "profile_step.py"} <= set(trees)
    bad = {name: list(_copies(tree)) for name, tree in trees.items() if name != "harness.py"}
    assert not {k: v for k, v in bad.items() if v}
    # the harness trips every construct check, so the check above is not passing on code it cannot see
    found = {what for _, what in _copies(trees["harness.py"])}
    assert {"constructs a CUDA graph", "constructs a timing event", "constructs torch.profiler.profile", "names nvidia-smi",
            "defines card", "defines timed", "defines graphed", "defines peak", "defines profile"} <= found


def test_stage_grouping_takes_the_first_stage_with_all_keys():
    stages = [("encoder attention", [("t5_attn", "<96")]), ("attention", [("t5_attn",)]),
              ("GEMMs and sums", [("tc_gemm",), ("colsum",)])]
    kernels = {"void grb::t5_attn_fwd<96>(Args)": (1500.0, 3), "void grb::t5_attn_fwd<64>(Args)": (700.0, 2),
               "void grb::tc_gemm<1>(Args)": (250.0, 9), "void grb::colsum_kernel(Args)": (50.0, 1),
               "Memcpy HtoD (Pageable -> Device)": (4.0, 1), "at::native::elementwise_kernel<add>": (6.0, 2)}
    split = harness.by_stage(kernels, stages, "torch")
    assert split == {"encoder attention": 1.5, "attention": 0.7, "GEMMs and sums": 0.3, "torch": 0.01}
    assert list(split) == ["encoder attention", "attention", "GEMMs and sums", "torch"]
    assert harness.mean_launch_us(kernels, "t5_attn") == 2200.0 / 5
    assert harness.largest_first(kernels, harness.short_name) == {
        "t5_attn_fwd<96>": 1500.0, "t5_attn_fwd<64>": 700.0, "tc_gemm<1>": 250.0, "colsum_kernel": 50.0,
        "at::native::elementwise_kernel<add>": 6.0, "Memcpy HtoD ": 4.0}


def _floor_plus_one(B, mean, lo, hi, g):
    """the HSTU and SASRec scripts' draw"""
    u = torch.rand(B, generator=g, dtype=torch.float64)
    return (torch.floor(torch.log1p(-u) / torch.log1p(torch.tensor(-1.0 / mean, dtype=torch.float64))) + 1).long().clamp(lo, hi)


def _ceil(B, mean, lo, hi, g):
    """the COBRA scripts' draw"""
    u = torch.rand(B, generator=g, dtype=torch.float64)
    return (torch.log1p(-u) / torch.log1p(torch.tensor(-1 / mean, dtype=torch.float64))).ceil().clamp(lo, hi).long()


# (old draw, B, mean, lo, hi) of every script that draws geometric lengths
DRAWS = [(_floor_plus_one, 128, 4, 1, 16), (_floor_plus_one, 128, 10, 1, 50), (_floor_plus_one, 1024, 9, 1, 50),
         (_floor_plus_one, 128, 9, 1, 50), (_floor_plus_one, 256, 9, 1, 50), (_ceil, 32, 9, 1, 20), (_ceil, 256, 9, 1, 20)]


@pytest.mark.parametrize("old,B,mean,lo,hi", DRAWS)
def test_geometric_lengths_reproduce_the_old_draws(old, B, mean, lo, hi):
    for seed in [0, 7, 1234] + list(range(1, 200)):
        a, b = torch.Generator().manual_seed(seed), torch.Generator().manual_seed(seed)
        new = harness.geometric_lengths(B, mean, lo, hi, a)
        assert new.dtype == torch.int64 and torch.equal(new, old(B, mean, lo, hi, b))
        assert torch.equal(a.get_state(), b.get_state())             # the same draws consumed: what follows is unchanged too


# the COBRA scripts' workloads in order, (B, items, texts), all drawn from one generator seeded 0
COBRA_RUNS = {"bench_cobra": [(32, "geometric", "short"), (32, "full", "full"), (256, "geometric", "short"), (256, "full", "full")],
              "bench_cobra_generate": [(32, "full", "full"), (32, "geometric", "full"), (256, "full", "full"), (256, "geometric", "full")]
              + [(32, "full", "full")] + [(256, "full", "full")] * 2,
              "bench_cobra_pool": [(256, "full", "full"), (32, "full", "full"), (256, "full", "full"), (256, "full", "full"),
                                   (256, "geometric", "full")]}


def test_geometric_lengths_at_the_scripts_generator_states():
    # bench_extend_jagged's cfg2_events: 128 of 4,096 users, uniform histories, then the geometric new items
    a, b = torch.Generator().manual_seed(7), torch.Generator().manual_seed(7)
    for g in (a, b):
        torch.randperm(4096, generator=g)
        torch.randint(1, 151, (128,), generator=g)
    assert torch.equal(harness.geometric_lengths(128, 4, 1, 16, a), _floor_plus_one(128, 4, 1, 16, b))
    for runs in COBRA_RUNS.values():
        a, b = torch.Generator().manual_seed(0), torch.Generator().manual_seed(0)
        for B, items, texts in runs:
            if items == "geometric":
                assert torch.equal(harness.geometric_lengths(B, 9, 1, 20, a), _ceil(B, 9, 1, 20, b))
            for g in (a, b):
                if texts == "short":
                    torch.randint(16, 65, (64,), generator=g)
                torch.randint(0, 1 << 30, (1,), generator=g)
