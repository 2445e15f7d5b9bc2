"""What the tools/bench_*.py scripts share: the card a number was taken on, CUDA-event and host timing, and the HBM
bandwidth their byte floors are computed against."""
import subprocess
import time

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet


def card():
    """'name, power limit, SM clock, max SM clock' of the first GPU, from a read-only nvidia-smi query; the device
    name torch reports where nvidia-smi cannot be run."""
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30, check=True)
        return q.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        import torch
        return torch.cuda.get_device_name()


def timed(fn, iters, warm=3):
    """(seconds per call, kernel launches per call) of `fn` over `iters` calls after `warm` calls, by CUDA events."""
    import torch
    from prysm_b200 import _ops
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    n0 = _ops.launch_count()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e-3 / iters, (_ops.launch_count() - n0) / iters


def host_time(fn):
    """Seconds of one call of `fn` on the host clock."""
    t0 = time.perf_counter()
    fn()
    return time.perf_counter() - t0
