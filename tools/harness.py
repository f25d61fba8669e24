"""What the model benchmarks in tools/ share: the hardware context of a run, the data-sheet HBM bandwidth their bounds
use, one kernel timer, bench.py's way of timing training steps and the launch list of one eager step.

The scripts put the repository's root on sys.path before they import this module."""
import subprocess

import bench

# NVIDIA's H100 SXM data sheet (700 W): HBM3 bandwidth, a ceiling, not a measurement
HBM_BYTES_PER_S = 3.35e12


def hardware():
    """Card name, power limit and max SM clock of cuda:0, read in the same run as the measurements."""
    import torch
    out = {"card": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        out["power_limit_w"] = float(q[0])
        out["max_sm_clock_mhz"] = float(q[1])
    except Exception as e:      # the numbers are then reported as unknown, never guessed
        out["power_limit_w"] = out["max_sm_clock_mhz"] = None
        out["query_error"] = repr(e)
    return out


def kernel_ms(fn, reps):
    """CUDA-event durations (ms) of ``reps`` calls of fn(), each waited for before the next, after one warm call."""
    import torch
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return ts


def time_train_steps(model, cfg, steps, warmup):
    """Train a compiled model on bench.py's synthetic batches of ``cfg`` as bench.py times it: at least ``warmup``
    steps, more until every batch has its step graph, then ``steps`` steps between two device events.  Raises if an
    id fell outside its table.  -> (ms per step, whether the steps were graph-replayed, the last step's summed loss)."""
    import torch
    dev = torch.device("cuda", 0)
    batches = [bench.device_inputs(cfg, x, y, dev) for x, y in bench.synth_batches(cfg, bench.N_BATCHES)]
    i = 0
    while i < warmup or (i < warmup + bench.N_BATCHES + 4 and model._graph_eligible()
                         and len(model._step_graphs) < bench.N_BATCHES):
        model.train_step(*batches[i % bench.N_BATCHES])
        i += 1
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for k in range(steps):
        loss = model.train_step(*batches[(i + k) % bench.N_BATCHES])
    e1.record()
    torch.cuda.synchronize()
    model._check_ids()
    return e0.elapsed_time(e1) / steps, bool(model._step_graphs), float(loss.item())


def launch_list(model, batch):
    """{wrapper name: {"launches", "ms"}} of one eager training step on ``batch`` (device features, labels), after
    one step to warm up."""
    from deepctr_b200 import kernels as K
    model.train_step(*batch)
    with K.profiled():
        model.train_step(*batch)
        prof = K.profile_summary()
    return {k: {"launches": n, "ms": round(ms, 4)} for k, (n, ms) in sorted(prof.items())}
