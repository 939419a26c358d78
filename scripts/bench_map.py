"""Time the `map` stage: the GPU CLI against the reference binary, on the configs[1] shape (100 Mbp genome, 30x, 150 bp PE FASTQ,
K = 63) by default.

Set-up, not timed: the reads are written to a private temporary directory, the graph is built by the GPU `pregraph` and the
reference's `contig`.  Timed: the GPU `map` (wall time, plus the stage's own split: CUDA-event times of the contig hash, the read
decode and the read scan, host times of the record pass and of the wait for the deflate) and the reference's `map` with -p equal to
the host's core count.  Both runs use the same -p, since -p is a layout parameter of .readInGap.gz.  Before any number is printed
the outputs are checked to be byte-identical.  Prints one JSON line, with the GPU's name and power limit read in the same run.

    python scripts/bench_map.py [--genome-len 100000000] [--coverage 30]
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
    a = ap.parse_args()
    import torch
    import bench
    from soapdenovo2_b200 import api
    ref_bin = os.path.join(ROOT, "oracle", "_ref", "SOAPdenovo-63mer")
    if not os.path.exists(ref_bin):
        raise SystemExit("oracle/_ref/SOAPdenovo-63mer is missing: run __graft_entry__.build() where the reference sources exist")
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the map stage is measured on the GPU only")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", os.environ.get("PGB200_DEVICE", "0")],
                         capture_output=True, text=True).stdout.strip()
    cores = os.cpu_count()
    d = tempfile.mkdtemp(prefix="pgb200_bench_map_")
    try:
        n_pairs = a.genome_len * a.coverage // 300
        t1, t2 = bench.gen_pe_fastq_gpu(torch, "cuda", a.genome_len, n_pairs, 42)
        t1.cpu().numpy().tofile(f"{d}/r_1.fq")
        t2.cpu().numpy().tofile(f"{d}/r_2.fq")
        del t1, t2
        torch.cuda.empty_cache()
        cfg = f"{d}/r.cfg"
        open(cfg, "w").write(f"max_rd_len=150\n[LIB]\navg_ins=300\nreverse_seq=0\nasm_flags=3\nrank=1\nq1={d}/r_1.fq\nq2={d}/r_2.fq\n")
        g = f"{d}/g"
        run([api.BIN63, "pregraph", "-s", cfg, "-K", str(a.K), "-p", "8", "-a", "16", "-R", "-o", g])
        run([ref_bin, "contig", "-g", g, "-R"])
        prefixes = {}
        for tag in ("gpu", "ref"):
            p = f"{d}/{tag}"
            for s in ("contig", "ContigIndex", "preGraphBasic"):
                shutil.copy(f"{g}.{s}", f"{p}.{s}")
            prefixes[tag] = p
        gpu_s, gpu_err = run([api.BIN63, "map", "-s", cfg, "-g", prefixes["gpu"], "-p", str(cores)], env=dict(os.environ, PGB200_VERBOSE="1"))
        ref_s, _ = run([ref_bin, "map", "-s", cfg, "-g", prefixes["ref"], "-p", str(cores)])
        bad = [s for s in ("readOnContig.gz", "readInGap.gz", "peGrads")
               if not filecmp.cmp(f"{prefixes['gpu']}.{s}", f"{prefixes['ref']}.{s}", shallow=False)]
        if bad:
            raise SystemExit(f"GPU map output differs from the reference's: {bad}")
        m = re.search(r"\[pgb200\] map: parse \.contig (\S+) ms \(host\), contig hash (\S+) ms, read decode (\S+) ms, read scan (\S+) ms "
                      r"\(GPU events\); reading (\S+) ms, record pass (\S+) ms, waiting for the deflate (\S+) ms", gpu_err)
        split = dict(zip(["parse_contig_ms_host", "contig_hash_ms_gpu", "read_decode_ms_gpu", "read_scan_ms_gpu", "reading_ms_host",
                          "record_pass_ms_host", "deflate_wait_ms_host"], map(float, m.groups()))) if m else None
        n_reads = 2 * n_pairs
        print(json.dumps({
            "metric": "map stage wall time", "unit": "s",
            "workload": f"synthetic {a.genome_len} bp genome, {a.coverage}x 150 bp PE FASTQ (insert 300), K={a.K}, {n_reads} reads",
            "gpu_map_s": round(gpu_s, 3), "gpu_split": split,
            "reference_map_s": round(ref_s, 3), "reference_threads": cores, "host_cores": cores,
            "outputs_identical": True, "gpu": gpu,
        }))
    finally:
        shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
