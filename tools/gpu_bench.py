"""What the avatar-creation benchmarks (bench_s3fd.py, bench_pfld.py, bench_bisenet.py) share: the card a number was measured on
and a CUDA-event timer."""
import subprocess


def gpu_info():
    """(name, power limit) of GPU 0 as nvidia-smi reports them; torch's device name and "unknown" without nvidia-smi."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, pl = [s.strip() for s in out.split(",")]
        return name, pl
    except Exception:
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def events_ms(fn, iters, warmup=0, stream=None):
    """Mean milliseconds per call of fn over iters calls, between two CUDA events on stream (torch's current stream if None),
    after warmup untimed calls and a device synchronise."""
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(iters):
        fn()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / iters
