"""Device time per view of every kernel of the bench workload's view-batch launches, from a torch.profiler trace.

bench.py's kernel_ms_per_view names kernels by their launch label, so the depth sort's onesweep passes and the tile sort's
both count as `sort_scatter` (and both histogram kernels as `sort_hist`).  Here the two sorts are told apart by grid size:
the depth sort runs ceil(P / 4096) blocks per view, the tile sort one block per 4096 instance slots.

    python tools/binning_profile.py [--steps 5] [--gaussians 1000000]

Runs bench.py's main() (no single-view leg, no CPU baseline) under torch.profiler with CUDA activities, keeps the kernels
whose grid has V rows (blockIdx.y = view: every launch of the batched step), and prints one JSON line: per kernel the summed
duration over (step count x V), where the step count is the number of batched render_fwd launches seen.  Kernels without a
view dimension are kept by name: tile_order (one block per view) and count_max (one thread).
"""
import argparse
import collections
import json
import math
import os
import re
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def short_name(name):
    name = re.sub(r"^void ", "", name)
    name = name.split("(")[0]
    name = re.sub(r"<.*>$", "", name)
    return name.split("::")[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    ap.add_argument("--views", type=int, default=8)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    sys.path.insert(0, ROOT)
    import bench
    sys.argv = ["bench.py", "--gpus", "1", "--steps", str(a.steps), "--warmup", "3", "--no-cpu-baseline", "--no-single-view",
                "--gaussians", str(a.gaussians), "--views-per-rank", str(a.views)]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        bench.main()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        events = json.load(open(path))["traceEvents"]

    depth_blocks = math.ceil(a.gaussians / (256 * 16))
    total = collections.defaultdict(float)
    count = collections.defaultdict(int)
    for e in events:
        if e.get("cat") != "kernel":
            continue
        grid = e.get("args", {}).get("grid", [0, 0, 0])
        n = short_name(e["name"])
        # tile_order runs one block per view (grid.x = V), count_max one thread
        batched = grid[1] == a.views or (n == "tile_order_kernel" and grid[0] == a.views) or n == "count_max_kernel"
        if not batched:
            continue
        if n in ("onesweep_pass_kernel", "onesweep_hist_kernel"):
            n += " (depth)" if grid[0] == depth_blocks else " (tile)"
        total[n] += e["dur"] / 1e3
        count[n] += 1
    steps = count.get("render_fwd_kernel", 0)
    if steps == 0:
        raise SystemExit("no batched render_fwd launch in the trace")
    per_view = {k: round(total[k] / (steps * a.views), 4) for k in sorted(total, key=lambda k: -total[k])}
    launches = {k: count[k] / steps for k in per_view}
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "steps_seen": steps, "views": a.views, "kernel_ms_per_view": per_view,
                      "launches_per_step": launches}), flush=True)


if __name__ == "__main__":
    main()
