"""Where the time of one pass 1 goes: the bench workload (bench.py's own generator and budget, configs[1] shape by default) fed from
HBM, warm-up steps, then timed steps under torch.profiler with CUDA activities.  Writes DIR/kernels.json (per-kernel GPU time per
step and launches per step, largest first, with the GPU's name and power limit) and DIR/trace.json (Chrome trace), and prints the
table.  PGB200_BUILD selects a variant build as everywhere else.

    python scripts/profile_pass1.py OUTDIR [--genome 100000000] [--K 63] [--steps 3] [--warmup 2]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--genome", type=int, default=100_000_000)
    ap.add_argument("--coverage", type=float, default=30.0)
    ap.add_argument("--K", type=int, default=63)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from soapdenovo2_b200 import api
    if not torch.cuda.is_available():
        raise SystemExit("profile_pass1.py needs a GPU")
    os.makedirs(args.outdir, exist_ok=True)
    dev = torch.device("cuda", 0)
    gpu = bench.gpu_identity(0)
    print(f"GPU: {gpu['name']}, power limit {gpu['power_limit_w']} W")
    budget = bench.per_gpu_budget(args.genome, args.coverage, args.K, 1, False, torch.cuda.get_device_properties(dev).total_memory)
    n_pairs = int(args.genome * args.coverage / (2 * bench.RD_LEN))
    t1, t2 = bench.gen_pe_fastq_gpu(torch, dev, args.genome, n_pairs, seed=42)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    eng = api.PregraphEngine(K=args.K, P=8, initG=0, flavour127=int(args.K > 63), max_rd_len=bench.RD_LEN, device=0, table_slots=budget["slots"])
    chunk = 4_000_000 * bench.REC_BYTES   # bench.py's device-resident feed: 4 M reads per feed_text call

    def step():
        eng.reset_pass1()
        for mate, t in enumerate((t1, t2)):
            for off in range(0, t.numel(), chunk):
                n = min(chunk, t.numel() - off)
                eng.feed_text(t.data_ptr() + off, n, on_device=True, fastq=True, ord_base=(off // bench.REC_BYTES) * 2 + mate, ord_stride=2)
        eng.finish_pass1()
        return eng.sweeps()

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
    prof.export_chrome_trace(os.path.join(args.outdir, "trace.json"))
    per = {}
    for ev in prof.events():
        if ev.device_type.name != "CUDA":
            continue
        d = per.setdefault(ev.name, [0.0, 0])
        d[0] += ev.time_range.elapsed_us() / 1e3   # a kernel's own duration, us -> ms
        d[1] += 1
    rows = sorted(({"kernel": k, "ms_per_step": v[0] / args.steps, "launches_per_step": v[1] / args.steps} for k, v in per.items()),
                  key=lambda r: -r["ms_per_step"])
    total = sum(r["ms_per_step"] for r in rows)
    out = {"gpu": gpu, "genome": args.genome, "coverage": args.coverage, "K": args.K, "steps": args.steps,
           "build": os.environ.get("PGB200_BUILD", ""), "gpu_ms_per_step": total, "kernels": rows}
    json.dump(out, open(os.path.join(args.outdir, "kernels.json"), "w"), indent=1)
    print(f"{'ms/step':>9} {'launches':>9}  kernel   (sum {total:.2f} ms of GPU time per step)")
    for r in rows[:25]:
        print(f"{r['ms_per_step']:9.2f} {r['launches_per_step']:9.1f}  {r['kernel'][:110]}")
    eng.close()


if __name__ == "__main__":
    main()
