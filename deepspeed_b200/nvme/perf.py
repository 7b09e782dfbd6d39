import argparse
import json
import os
import time

import torch


def run_io_benchmark(path, size_bytes, read=True, block_size=1 << 20, queue_depth=32, threads=1, single_submit=False,
                     overlap_events=True, loops=3, use_gds=False, device="cpu", validate=False):
    """Time ``loops`` whole-file reads or writes through the aio (or GDS) handle; returns GB/s stats."""
    from deepspeed_b200.ops.aio import aio_handle
    if use_gds:
        from deepspeed_b200.ops.gds import gds_handle
        h = gds_handle(block_size, queue_depth, single_submit, overlap_events, threads)
    else:
        h = aio_handle(block_size, queue_depth, single_submit, overlap_events, threads)
    n = size_bytes
    if device == "cpu":
        buf = h.new_cpu_locked_tensor(n, torch.empty(0, dtype=torch.uint8))
    else:
        buf = torch.empty(n, dtype=torch.uint8, device=device)
        if use_gds:
            h.pin_device_tensor(buf)
    if not read:
        buf.random_(0, 255) if device == "cpu" else buf.fill_(7)
    elif not os.path.exists(path) or os.path.getsize(path) < n:
        tmp = torch.randint(0, 255, (n, ), dtype=torch.uint8)
        h.sync_pwrite(tmp if device == "cpu" else tmp, path)
    times = []
    for _ in range(loops):
        t = time.perf_counter()
        if read:
            h.pread(buf, path, False, False, 0)
        else:
            h.pwrite(buf, path, False, False, 0)
        if device != "cpu":
            torch.cuda.synchronize()
        times.append(time.perf_counter() - t)
    if validate and read:
        ref = torch.empty(n, dtype=torch.uint8)
        with open(path, "rb") as f:
            ref = torch.frombuffer(bytearray(f.read(n)), dtype=torch.uint8)
        assert torch.equal(ref, buf.cpu()), "aio read validation failed"
    if device == "cpu":
        h.free_cpu_locked_tensor(buf)
    gbs = [n / t / 1e9 for t in times]
    return {"op": "read" if read else "write", "bytes": n, "block_size": block_size, "queue_depth": queue_depth,
            "threads": threads, "single_submit": single_submit, "overlap_events": overlap_events, "gds": use_gds,
            "gb_per_s_max": max(gbs), "gb_per_s_mean": sum(gbs) / len(gbs), "sec_min": min(times)}


def _parse_size(s):
    s = str(s).upper()
    for suf, m in (("G", 1 << 30), ("M", 1 << 20), ("K", 1 << 10)):
        if s.endswith(suf):
            return int(float(s[:-1]) * m)
    return int(s)


def ds_io_main(argv=None):
    p = argparse.ArgumentParser(description="DeepSpeed-H100 NVMe I/O benchmark")
    p.add_argument("--folder", "--nvme_dir", dest="folder", type=str, required=True)
    p.add_argument("--io_size", type=str, default="256M")
    p.add_argument("--read", action="store_true")
    p.add_argument("--block_size", type=str, default="1M")
    p.add_argument("--queue_depth", type=int, default=32)
    p.add_argument("--io_parallel", "--threads", dest="threads", type=int, default=1)
    p.add_argument("--single_submit", action="store_true")
    p.add_argument("--sequential_requests", dest="overlap_events", action="store_false")
    p.add_argument("--loops", type=int, default=3)
    p.add_argument("--use_gds", action="store_true")
    p.add_argument("--gpu", action="store_true")
    p.add_argument("--validate", action="store_true")
    a = p.parse_args(argv)
    os.makedirs(a.folder, exist_ok=True)
    r = run_io_benchmark(os.path.join(a.folder, "ds_io_test.bin"), _parse_size(a.io_size), a.read, _parse_size(a.block_size),
                         a.queue_depth, a.threads, a.single_submit, a.overlap_events, a.loops, a.use_gds,
                         "cuda" if a.gpu else "cpu", a.validate)
    print(json.dumps(r))
    return r
