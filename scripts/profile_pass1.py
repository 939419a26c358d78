"""Where the time of one pass 1 goes: the bench workload (bench.py's own generator and budget, configs[1] shape by default) fed from
HBM, warm-up steps, then timed steps under torch.profiler with CUDA activities.  Writes DIR/kernels.json (per-kernel GPU time per
step and launches per step, largest first, with the GPU's name and power limit) and DIR/trace.json (Chrome trace), and prints the
table.  Per timed step it also prints the front-end span (first GPU activity of the step -> start of k_skm_apply) and, inside that
span, every stream's busy time and the idle time between its activities.  The per-kernel sums add up durations of kernels that share
the SMs; run once more with CUDA_LAUNCH_BLOCKING=1 for each kernel's time with nothing beside it.  PGB200_BUILD selects a variant
build as everywhere else.

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
    from torch.profiler import ProfilerActivity, profile, record_function
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
            with record_function(STEP_MARK):
                step()
        torch.cuda.synchronize()
    prof.export_chrome_trace(os.path.join(args.outdir, "trace.json"))
    spans = step_spans(json.load(open(os.path.join(args.outdir, "trace.json"))))
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
           "build": os.environ.get("PGB200_BUILD", ""), "launch_blocking": os.environ.get("CUDA_LAUNCH_BLOCKING", "0"),
           "gpu_ms_per_step": total, "kernels": rows, "steps_front_end": spans}
    json.dump(out, open(os.path.join(args.outdir, "kernels.json"), "w"), indent=1)
    print(f"{'ms/step':>9} {'launches':>9}  kernel   (sum {total:.2f} ms of GPU time per step)")
    for r in rows[:25]:
        print(f"{r['ms_per_step']:9.2f} {r['launches_per_step']:9.1f}  {r['kernel'][:110]}")
    for i, s in enumerate(spans):
        print(f"step {i}: front end {s['front_end_ms']:.2f} ms (first GPU activity -> start of k_skm_apply), apply {s['apply_ms']:.2f} ms")
        for st in s["streams"]:
            print(f"    stream {st['stream']:>3} ({st['role']:>9}): busy {st['busy_ms']:7.2f} ms, idle between its activities {st['gap_ms']:7.2f} ms, "
                  f"first activity at +{st['first_ms']:.2f} ms")
            for k, v in st["kernels"][:6]:
                print(f"        {v:7.2f} ms  {k[:100]}")
    eng.close()


STEP_MARK = "pass1_step"
GPU_CATS = ("kernel", "gpu_memset", "gpu_memcpy")


def _union_ms(iv):
    """Length of the union of [start, end) intervals (us), in ms."""
    tot, cur_s, cur_e = 0.0, None, None
    for s, e in sorted(iv):
        if cur_e is None or s > cur_e:
            if cur_e is not None:
                tot += cur_e - cur_s
            cur_s, cur_e = s, e
        else:
            cur_e = max(cur_e, e)
    if cur_e is not None:
        tot += cur_e - cur_s
    return tot / 1e3


def step_spans(trace):
    """Per timed step, from the Chrome trace: the front-end span (first GPU activity of the step -> start of the k_skm_apply launch) and,
    inside it, every stream's busy time (union of its activities), the idle time between its activities, and its kernels.  A step's GPU
    work lies inside the host range of its record_function: it is launched there, and the step ends by reading results back."""
    evs = trace["traceEvents"] if isinstance(trace, dict) else trace
    marks = sorted((e["ts"], e["ts"] + e["dur"]) for e in evs if e.get("ph") == "X" and e.get("cat") == "user_annotation" and e.get("name") == STEP_MARK)
    gpu = [e for e in evs if e.get("ph") == "X" and e.get("cat") in GPU_CATS]
    out = []
    for m0, m1 in marks:
        acts = sorted((e for e in gpu if m0 <= e["ts"] < m1), key=lambda e: e["ts"])
        apply = [e for e in acts if "k_skm_apply" in e["name"]]
        if not acts or not apply:
            continue
        t0, t_apply = acts[0]["ts"], apply[0]["ts"]
        streams = {}
        for e in acts:
            if e["ts"] >= t_apply:
                continue
            sid = e.get("args", {}).get("stream", e.get("tid"))
            streams.setdefault(sid, []).append(e)
        rows = []
        for sid, es in streams.items():
            iv = [(e["ts"], min(e["ts"] + e["dur"], t_apply)) for e in es]
            busy = _union_ms(iv)
            names = " ".join(e["name"] for e in es)
            role = ("partition" if "k_skm_count" in names else "decode" if "k_decode_fast" in names
                    else "clear" if any(e["cat"] == "gpu_memset" and e["dur"] > 1000 for e in es) else "other")
            per_k = {}
            for e in es:
                per_k[e["name"]] = per_k.get(e["name"], 0.0) + min(e["dur"], t_apply - e["ts"]) / 1e3
            rows.append({"stream": sid, "role": role, "busy_ms": busy, "first_ms": (iv[0][0] - t0) / 1e3,
                         "gap_ms": (max(e for _, e in iv) - iv[0][0]) / 1e3 - busy,
                         "kernels": sorted(per_k.items(), key=lambda kv: -kv[1])})
        rows.sort(key=lambda r: -r["busy_ms"])
        out.append({"front_end_ms": (t_apply - t0) / 1e3, "apply_ms": apply[0]["dur"] / 1e3, "streams": rows})
    return out


if __name__ == "__main__":
    main()
