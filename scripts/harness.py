"""What the benchmark scripts share: the card a number was measured on, eager and CUDA-graph timing with CUDA events, peak memory,
one torch.profiler run and its views, and the seeded workload draws.  Imported by the scripts, never run itself."""
import subprocess

import torch
from torch.profiler import ProfilerActivity


def card(device="cuda"):
    """The device's name, power limit and max SM clock, read now: an absolute number is only worth something beside them.  The
    card is queried by its UUID, since CUDA's device order and CUDA_VISIBLE_DEVICES need not match nvidia-smi's indices."""
    index = torch.device(device).index
    index = torch.cuda.current_device() if index is None else index
    uuid = str(torch.cuda.get_device_properties(index).uuid)
    uuid = uuid if uuid.startswith(("GPU-", "MIG-")) else "GPU-" + uuid
    try:
        r = subprocess.run(["nvidia-smi", "-i", uuid, "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        q = r.stdout.strip() if r.returncode == 0 else ""
    except (OSError, subprocess.SubprocessError):
        q = ""
    return dict(gpu=torch.cuda.get_device_name(index), power_limit_and_max_sm_clock=q or "unknown")


def timed(fn, steps, warmup):
    """(ms per call, peak bytes allocated) of `steps` calls of fn between CUDA events, after `warmup` untimed calls"""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / steps, torch.cuda.max_memory_allocated()


def graphed(fn, warmup, calls=1):
    """(graph, output of its last call) of `calls` calls of fn captured in one CUDA graph, after `warmup` calls on a side stream.
    Each call's output is dropped before the next, so the calls share one set of output buffers.  Time the graph with
    timed(graph.replay, steps, 1)."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(warmup):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(calls - 1):
            fn()
        out = fn()
    return graph, out


def peak(fn):
    """peak bytes allocated during one call of fn (the caller subtracts its own baseline)"""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated()


def profile(fn, calls=1, warmup=1, cpu=False):
    """{name: (device us, count)} of everything with device time in one torch.profiler run over `calls` calls of fn, after `warmup`
    untimed ones: each kernel with its launches.  cpu=True also records the CPU ops and record_function ranges, each with the device
    time of the kernels it launched."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    activities = [ProfilerActivity.CUDA] + ([ProfilerActivity.CPU] if cpu else [])
    with torch.profiler.profile(activities=activities) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    return {e.key: (e.device_time_total, e.count) for e in prof.key_averages() if e.device_time_total > 0}


def short_name(name, cut="("):
    """a kernel's name without its arguments (cut="<": without its template arguments too), `void ` and the `grb::` namespace"""
    return name.split(cut)[0].replace("void ", "").replace("grb::", "")


def largest_first(kernels, name=lambda k: k):
    """{name(kernel): us} of a profile, summed over kernels of one name, largest first"""
    out = {}
    for k, (us, _) in kernels.items():
        out[name(k)] = out.get(name(k), 0.0) + us
    return dict(sorted(out.items(), key=lambda kv: -kv[1]))


def by_stage(kernels, stages, other):
    """{stage: ms} of a profile, largest first.  stages: [(stage, [keys, ...]), ...]; a kernel belongs to the first stage with a
    tuple of keys that are all in its name, else to `other`."""
    out = {}
    for k, (us, _) in kernels.items():
        stage = next((s for s, alts in stages if any(all(key in k for key in keys) for keys in alts)), other)
        out[stage] = out.get(stage, 0.0) + us / 1000.0
    return {s: round(ms, 2) for s, ms in sorted(out.items(), key=lambda kv: -kv[1])}


def mean_launch_us(kernels, part):
    """mean device us per launch of the kernels whose name contains `part` (nan if none ran)"""
    hits = [v for k, v in kernels.items() if part in k]
    total, count = sum(us for us, _ in hits), sum(n for _, n in hits)
    return total / count if count else float("nan")


def geometric_lengths(B, mean, lo, hi, generator):
    """B lengths geometric on 1, 2, ... with the given mean, clamped to [lo, hi], drawn by inversion from one float64 uniform each"""
    u = torch.rand(B, generator=generator, dtype=torch.float64)
    x = torch.log1p(-u) / torch.log1p(torch.tensor(-1 / mean, dtype=torch.float64))
    return (torch.floor(x) + 1).long().clamp(lo, hi)


def cobra_batch(B, items, g, texts="full"):
    """(input_ids, encoder_input_ids) of B COBRA users at the trainer's shape, drawn from g: every user at 20 items (items="full")
    or item counts geometric with mean 9 capped at 20; texts of 128 tokens (texts="full") or 64 lengths uniform on [16, 64]"""
    from tests import cobra_params as cp
    n = [20] * B if items == "full" else geometric_lengths(B, 9, 1, 20, g).tolist()
    lens = [128] if texts == "full" else torch.randint(16, 65, (64,), generator=g).tolist()
    return cp.batch(cp.TRAINER, items=n, text_lens=lens, L=128, seed=int(torch.randint(0, 1 << 30, (1,), generator=g)))
