#!/usr/bin/env python
"""bench_sharded.py — what a document-sharded index costs on the C3 workload (bench.py's corpus and query seeds).

End to end through host buffers (bm25x_search_batch / bm25x_sharded_search_batch from page-locked host arrays, results
back to the host every step): the unsharded index against S = 1, 2 and 4 shards on one GPU, the arms alternating step by
step, `--steps` timed steps per arm after `--warmup`.  Every arm's rows must be identical to the unsharded index's.  The
merge kernel (k_merge_shards) is timed on its own with torch.profiler over one extra step per sharded arm.  With two GPUs
visible, an S = 2 arm with one shard per device is added.  Prints one JSON line; writes nothing.

  python tools/bench_sharded.py [--steps 20] [--warmup 3] [--docs N] [--queries Q] [--k 10]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,power.max_limit",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit, max_limit = [x.strip() for x in out.split(",")[:3]]
        return {"name": name, "power_limit": limit, "power_max_limit": max_limit}
    except Exception as e:  # noqa: BLE001 — reported in the output
        return {"error": str(e)}


def merge_kernel_ms(torch, run):
    """Device time of k_merge_shards during one call of `run`, from torch.profiler's CUDA activity."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    total = 0.0
    for ev in prof.events():
        if "k_merge_shards" in ev.name:
            t = getattr(ev, "device_time_total", None)
            total += (t if t is not None else ev.cuda_time_total) / 1e3
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--queries", type=int, default=100_000)
    ap.add_argument("--k", type=int, default=10)
    a = ap.parse_args()
    import torch

    import _pkg
    m = _pkg.load()
    m.load_library()
    seed, vocab, k, nq = 0xB25C0DE0 + 3, 100_000, a.k, a.queries      # bench.py WORKLOADS["c3"]
    t0 = time.time()
    c = m.synth_corpus(seed, a.docs, vocab, 128, 128, 0.0)
    q_off, q_terms = m.synth_queries(seed + 1000, nq, vocab, 3, 3, c.post_off)
    t_gen = time.time() - t0

    def pinned(shape, dtype, src=None):
        n = int(np.prod(shape)) * np.dtype(dtype).itemsize
        buf = torch.empty(max(n, 1), dtype=torch.uint8, pin_memory=True).numpy()[:n].view(dtype).reshape(shape)
        if src is not None:
            buf[...] = src
        return buf

    q_off, q_terms = pinned(q_off.shape, np.uint32, q_off), pinned(q_terms.shape, np.uint32, q_terms)
    arms, build_s = {}, {}
    t0 = time.time()
    arms["unsharded"] = m.Index.from_corpus(c)
    build_s["unsharded"] = time.time() - t0
    plan = [(1, None), (2, None), (4, None)]
    if m.device_count() >= 2:
        plan.append((2, [0, 1]))
    for S, devs in plan:
        name = f"S={S}" + (" on devices 0,1" if devs else "")
        t0 = time.time()
        arms[name] = m.ShardedIndex.from_corpus(c, n_shards=S, devices=devs)
        build_s[name] = time.time() - t0
    outs = {name: {"doc": pinned((nq, k), np.uint32), "score": pinned((nq, k), np.float32),
                   "score64": pinned((nq, k), np.float64), "payload": None, "n": pinned((nq,), np.uint32)}
            for name in arms}
    times = {name: [] for name in arms}
    kernel_ms = {name: [] for name in arms}
    for step in range(a.warmup + a.steps):
        for name, idx in arms.items():   # alternating: drift of clocks or neighbours hits every arm alike
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = idx.search_batch(q_off, q_terms, k, out=outs[name])
            dt = time.perf_counter() - t0
            if step >= a.warmup:
                times[name].append(dt)
                kernel_ms[name].append(r["stats"].kernel_ms)
    ref = outs["unsharded"]
    identical = {name: all(np.array_equal(o[key], ref[key]) for key in ("doc", "score", "score64", "n"))
                 for name, o in outs.items()}
    merge_ms = {name: merge_kernel_ms(torch, lambda idx=idx, name=name: idx.search_batch(q_off, q_terms, k, out=outs[name]))
                for name, idx in arms.items() if name != "unsharded"}
    base = statistics.median(times["unsharded"])
    result = {"metric": "sharded vs unsharded index, C3 end to end through host buffers (queries/s)",
              "workload": f"C3: {a.docs} docs, vocab {vocab} uniform, 128 terms/doc, {nq} 3-term queries, top-{k}",
              "steps": a.steps, "warmup": a.warmup, "card": card(), "gen_s": round(t_gen, 1),
              "arms": {name: {"qps": nq / statistics.median(times[name]), "ms_median": 1e3 * statistics.median(times[name]),
                              "ms_min": 1e3 * min(times[name]), "vs_unsharded": base / statistics.median(times[name]),
                              "kernel_ms_summed": statistics.median(kernel_ms[name]),
                              "merge_kernel_ms": merge_ms.get(name), "build_s": round(build_s[name], 1),
                              "device_bytes": int(idx.info().device_bytes), "identical": identical[name]}
                       for name, idx in arms.items()},
              "note": "kernel_ms_summed is device time summed over the shards and the merge, not wall time"}
    print(json.dumps(result))
    for idx in arms.values():
        idx.close()
    if not all(identical.values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
