"""Time the long-read pass of the `map` stage (asm_flags=4, k_map_long) against the reference, on the bench_map.py graph (the
configs[1] shape by default: 100 Mbp genome, 30x 150 bp PE FASTQ, K = 63) plus seeded long reads of 1-10 kbp (about 1 Gbp by
default) in a library with rd_len_cutoff=10000.

Set-up, not timed: the reads are written to a private temporary directory, the graph is built by the GPU `pregraph` and the
reference's `contig`.  Timed: the GPU `map` with PGB200_VERBOSE (the long pass's wall time and its CUDA-event scan time) and the
reference's `map` at the same -p (16 by default; its `Time spent on aligning long reads`, whole seconds).  The outputs are
checked to be byte-identical, .longReadInGap included, before any number is printed.  Lookups per second are set against the HBM
random-access bound of one 32 B sector per lookup.  Prints one JSON line, with the GPU's name and power limit read in the same run.

    python scripts/bench_map_long.py [--genome-len 100000000] [--coverage 30] [--long-gbp 1.0]
"""
import argparse
import filecmp
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12   # H100 SXM5 80 GB HBM3 peak


def run(cmd, env=None):
    t = time.perf_counter()
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    dt = time.perf_counter() - t
    if r.returncode != 0:
        raise SystemExit(f"{' '.join(cmd)} failed ({r.returncode}):\n{r.stderr[-3000:]}")
    return dt, r.stderr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genome-len", type=int, default=100_000_000)
    ap.add_argument("--coverage", type=int, default=30)
    ap.add_argument("--K", type=int, default=63)
    ap.add_argument("--long-gbp", type=float, default=1.0)
    ap.add_argument("--threads", type=int, default=16, help="-p of both runs (a layout parameter of .longReadInGap)")
    a = ap.parse_args()
    import torch
    import bench
    from soapdenovo2_b200 import api, synth
    ref_bin = os.path.join(ROOT, "oracle", "_ref", "SOAPdenovo-63mer")
    if not os.path.exists(ref_bin):
        raise SystemExit("oracle/_ref/SOAPdenovo-63mer is missing: run __graft_entry__.build() where the reference sources exist")
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the map stage is measured on the GPU only")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", os.environ.get("PGB200_DEVICE", "0")],
                         capture_output=True, text=True).stdout.strip()
    d = tempfile.mkdtemp(prefix="pgb200_bench_map_long_")
    try:
        n_pairs = a.genome_len * a.coverage // 300
        t1, t2 = bench.gen_pe_fastq_gpu(torch, "cuda", a.genome_len, n_pairs, 42)
        t1.cpu().numpy().tofile(f"{d}/r_1.fq")
        t2.cpu().numpy().tofile(f"{d}/r_2.fq")
        del t1, t2
        genome, _ = bench.gen_genome(torch, "cuda", a.genome_len, 42)   # the same genome the paired reads come from
        g_host = genome.cpu().numpy()
        del genome
        torch.cuda.empty_cache()
        n_long = max(2, int(a.long_gbp * 1e9 / 5500))
        reads = synth.long_reads(g_host, n_long, 1000, 10000, seed=7, short_frac=0.0)
        synth.write_long(f"{d}/long.fa", reads, fastq=False)
        long_bases = sum(len(r) for r in reads)
        del reads, g_host
        cfg = f"{d}/r.cfg"
        open(cfg, "w").write(f"max_rd_len=150\n[LIB]\navg_ins=300\nreverse_seq=0\nasm_flags=3\nrank=1\nq1={d}/r_1.fq\nq2={d}/r_2.fq\n"
                             f"[LIB]\nasm_flags=4\nrd_len_cutoff=10000\nmap_len=40\nf={d}/long.fa\n")
        g = f"{d}/g"
        run([api.BIN63, "pregraph", "-s", cfg, "-K", str(a.K), "-p", "8", "-a", "16", "-R", "-o", g])
        run([ref_bin, "contig", "-g", g, "-R"])
        prefixes = {}
        for tag in ("gpu", "ref"):
            p = f"{d}/{tag}"
            for s in ("contig", "ContigIndex", "preGraphBasic"):
                shutil.copy(f"{g}.{s}", f"{p}.{s}")
            prefixes[tag] = p
        P = str(a.threads)
        gpu_s, gpu_err = run([api.BIN63, "map", "-s", cfg, "-g", prefixes["gpu"], "-p", P], env=dict(os.environ, PGB200_VERBOSE="1"))
        ref_s, ref_err = run([ref_bin, "map", "-s", cfg, "-g", prefixes["ref"], "-p", P])
        bad = [s for s in ("longReadInGap", "readOnContig.gz", "readInGap.gz", "peGrads")
               if not filecmp.cmp(f"{prefixes['gpu']}.{s}", f"{prefixes['ref']}.{s}", shallow=False)]
        if bad:
            raise SystemExit(f"GPU map output differs from the reference's: {bad}")
        m = re.search(r"\[pgb200\] map long pass: (\d+) reads, (\S+) ms \(host\), long-read scan (\S+) ms \(GPU events\), (\d+) lookups", gpu_err)
        ref_long = re.search(r"Time spent on aligning long reads: (\d+)s", ref_err)
        n_reads, long_wall_ms, scan_ms, lookups = int(m.group(1)), float(m.group(2)), float(m.group(3)), int(m.group(4))
        lookups_per_s = lookups / (scan_ms * 1e-3) if scan_ms > 0 else None
        print(json.dumps({
            "metric": "map long-read pass", "unit": "ms",
            "workload": f"synthetic {a.genome_len} bp genome, {a.coverage}x 150 bp PE FASTQ (insert 300), K={a.K}; {n_reads} long reads "
                        f"of 1-10 kbp ({long_bases} bases, 1% errors), rd_len_cutoff=10000, map_len=40",
            "gpu_long_scan_ms_events": scan_ms, "gpu_long_pass_ms_wall": long_wall_ms, "gpu_map_s": round(gpu_s, 3),
            "lookups": lookups, "lookups_per_s": lookups_per_s,
            "hbm_bound_lookups_per_s": HBM_BYTES_PER_S / 32, "fraction_of_hbm_bound": lookups_per_s / (HBM_BYTES_PER_S / 32) if lookups_per_s else None,
            "reference_long_pass_s": int(ref_long.group(1)) if ref_long else None, "reference_map_s": round(ref_s, 3), "threads": a.threads,
            "host_cores": os.cpu_count(), "outputs_identical": True, "gpu": gpu,
        }))
    finally:
        shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
