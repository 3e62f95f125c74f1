#!/usr/bin/env python3
"""Experiment: is the C2 throughput (bench.py's resident arm) bounded by what the host threads can submit, or by the GPU?

    python scripts/exp_submit_rate.py [--handles 8,16] [--steps 40] [--warmup 5] [--out DIR]

For each handle count S: S host threads, one Core each, `steps` vgicp_register calls per thread on distinct resident pairs of a pool
larger than the L2 (bench.py's protocol).  Reports registrations/s (device time from a common start event to the last stream's end
event), host CPU time per registration (time.thread_time in every worker) and kernel launches per registration.  A second, separate
pass records a few steps with torch.profiler (CUDA activities) and reports from its trace the GPU busy fraction -- the union of all
kernel intervals over the window from the first to the last kernel -- and the CUDA runtime calls per registration by name.
The trace is written under DIR.  VGICP_B200_LIB selects another build of the library (A/B comparisons).
"""
import argparse
import json
import os
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")


def busy_fraction(trace_path):
    ev = json.load(open(trace_path))
    ev = ev["traceEvents"] if isinstance(ev, dict) else ev
    kern = sorted((e["ts"], e["ts"] + e["dur"]) for e in ev if e.get("cat") == "kernel" and "dur" in e)
    calls = {}
    for e in ev:
        if e.get("cat") in ("cuda_runtime", "cuda_driver"):
            calls[e["name"]] = calls.get(e["name"], 0) + 1
    if not kern:
        return None, 0.0, calls, 0
    busy, cur_s, cur_e = 0.0, kern[0][0], kern[0][1]
    for s, e in kern[1:]:
        if s > cur_e:
            busy += cur_e - cur_s
            cur_s, cur_e = s, e
        else:
            cur_e = max(cur_e, e)
    busy += cur_e - cur_s
    span = kern[-1][1] - kern[0][0]
    return busy / span, span * 1e-3, calls, len(kern)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--handles", default="8,16")
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile-steps", type=int, default=4)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "exp_submit_rate"), help="directory for the traces and the JSON record")
    ap.add_argument("--tag", default="")
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)

    import torch
    from torch.profiler import ProfilerActivity, profile

    from fast_gicp_b200.core import LIB_PATH, REG_PLANE, Core

    dev = torch.device("cuda", 0)
    d = np.load(os.path.join(ROOT, "tests", "golden", "pair_0p1.npz"))
    tgt, src = np.ascontiguousarray(d["target"], np.float32), np.ascontiguousarray(d["source"], np.float32)
    n_t, n_s = len(tgt), len(src)
    P = int(np.ceil(160e6 / ((n_t + n_s) * 12)))
    rng = np.random.default_rng(1234)
    t0, s0 = torch.from_numpy(tgt).to(dev), torch.from_numpy(src).to(dev)
    pool_t = torch.empty((P, n_t, 3), dtype=torch.float32, device=dev)
    pool_s = torch.empty((P, n_s, 3), dtype=torch.float32, device=dev)
    for i in range(P):
        yaw = rng.uniform(-0.05, 0.05) if i else 0.0
        R = torch.tensor([[np.cos(yaw), -np.sin(yaw), 0.0], [np.sin(yaw), np.cos(yaw), 0.0], [0.0, 0.0, 1.0]], dtype=torch.float32, device=dev)
        t = torch.tensor(rng.uniform(-0.5, 0.5, size=3) * (1.0 if i else 0.0), dtype=torch.float32, device=dev)
        pool_t[i] = t0 @ R.T + t
        pool_s[i] = s0 @ R.T + t
    torch.cuda.synchronize()
    tp, sp = pool_t.data_ptr(), pool_s.data_ptr()
    props = torch.cuda.get_device_properties(0)
    record = {"lib": LIB_PATH, "tag": args.tag, "gpu": props.name, "pool_pairs": P, "runs": []}
    try:
        import subprocess

        record["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:  # noqa: BLE001
        record["power_limit"] = repr(e)

    for S in [int(x) for x in args.handles.split(",")]:
        cores = [Core(0) for _ in range(S)]
        for c in cores:
            c.set_resolution(1.0)
            c.set_neighbor_search_method("DIRECT27")
            c.set_execution_hint(0)
        streams = [torch.cuda.ExternalStream(c.stream(), device=dev) for c in cores]

        def run(steps):
            start = torch.cuda.Event(enable_timing=True)
            ends = [torch.cuda.Event(enable_timing=True) for _ in range(S)]
            cpu = [0.0] * S
            start_barrier = threading.Barrier(S + 1)

            def work(ci):
                start_barrier.wait()
                c0 = time.thread_time()
                for j in range(steps):
                    pi = (ci + j * S) % P
                    cores[ci].register_raw(tp + pi * n_t * 12, n_t, sp + pi * n_s * 12, n_s, 12, True, 20, REG_PLANE)
                cpu[ci] = time.thread_time() - c0
                ends[ci].record(streams[ci])

            th = [threading.Thread(target=work, args=(ci,)) for ci in range(S)]
            for t_ in th:
                t_.start()
            torch.cuda.synchronize()
            start.record(torch.cuda.current_stream())
            torch.cuda.current_stream().synchronize()
            w0 = time.perf_counter()
            start_barrier.wait()
            for t_ in th:
                t_.join()
            torch.cuda.synchronize()
            return max(start.elapsed_time(e) for e in ends), time.perf_counter() - w0, sum(cpu)

        run(args.warmup)
        l0 = sum(c.launch_count() for c in cores)
        ms, wall, cpu = run(args.steps)
        launches = sum(c.launch_count() for c in cores) - l0
        regs = S * args.steps
        rec = {"handles": S, "registrations": regs, "registrations_per_s": regs / (ms * 1e-3), "wall_registrations_per_s": regs / wall,
               "host_cpu_ms_per_registration": 1e3 * cpu / regs, "host_threads_cpu_busy": cpu / (S * wall), "launches_per_registration": launches / regs}
        # separate traced pass
        trace = os.path.join(args.out, "trace_%s_h%d.pt.trace.json" % (args.tag or "run", S))
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            run(args.profile_steps)
        prof.export_chrome_trace(trace)
        frac, span_ms, calls, nk = busy_fraction(trace)
        pr = S * args.profile_steps
        rec.update(gpu_busy_fraction=frac, traced_span_ms=span_ms, traced_kernels_per_registration=nk / pr,
                   runtime_calls_per_registration={k: v / pr for k, v in sorted(calls.items(), key=lambda kv: -kv[1])},
                   runtime_calls_per_registration_total=sum(calls.values()) / pr)
        record["runs"].append(rec)
        print(json.dumps(rec), flush=True)
        for c in cores:
            c.close()
    with open(os.path.join(args.out, "submit_rate_%s.json" % (args.tag or "run")), "w") as f:
        json.dump(record, f, indent=1)


if __name__ == "__main__":
    main()
