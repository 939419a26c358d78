"""Measure the GPU gzip writer (soapdenovo2_b200/csrc/deflate.cu) and what it does to the stages.

  1. Writer throughput on `.readOnContig`-shaped and `.edge`-shaped text: the GPU writer's input GB/s (device-resident and
     host-resident input, open to close) and zlib's gzwrite MB/s on the same text (PGB200_GZ=host).  Every GPU file is checked
     against zlib's bytes before its number is printed.
  2. `pregraph` (-R, .edge.gz written) and `map` wall time on the configs[1] shape (100 Mbp genome, 30x 150 bp PE FASTQ, K = 63),
     with PGB200_GZ=gpu and with PGB200_GZ=host, with the stage's PGB200_VERBOSE split; the two runs' files are compared.
     Set-up (reads, the reference's `contig` for the map graph) is not timed.  --skip-stages leaves part 2 out.

Prints one JSON line, with the GPU's name and power limit read in the same run.

    python scripts/bench_gzip.py [--mb 512] [--genome-len 100000000] [--coverage 30] [--skip-stages]
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
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def run(cmd, env):
    t = time.perf_counter()
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    dt = time.perf_counter() - t
    if r.returncode != 0:
        raise SystemExit(f"{' '.join(cmd)} failed ({r.returncode}):\n{r.stderr[-3000:]}")
    return dt, r.stderr


def text(kind, n):
    import numpy as np
    rng = np.random.default_rng(5)
    if kind == "read_on_contig":
        m = n // 20 + 1
        cols = [np.arange(1, m + 1), rng.integers(1, 2_000_000, m), rng.integers(0, 30000, m)]
        ori = np.where(rng.integers(0, 2, m) == 1, "+", "-")
        return "".join(f"{a}\t{b}\t{c}\t{d}\n" for a, b, c, d in zip(*(c.tolist() for c in cols), ori.tolist())).encode()[:n]
    out = []   # .edge: a header line per edge, then its bases in 100-column lines
    size = 0
    acgt = np.frombuffer(b"ACGT", np.uint8)
    while size < n:
        L = int(rng.integers(64, 2000))
        seq = acgt[rng.integers(0, 4, L + 62)].tobytes()
        rec = (b">length %d,%d,%d,%d,%d\n" % (L, rng.integers(1 << 30), rng.integers(1 << 30), rng.integers(-1, 2), rng.integers(1, 60))
               + b"".join(seq[j:j + 100] + b"\n" for j in range(0, len(seq), 100)))
        out.append(rec)
        size += len(rec)
    return b"".join(out)[:n]


def writer_numbers(mb, d):
    import torch
    from soapdenovo2_b200 import api
    res = {}
    for kind in ("read_on_contig", "edge"):
        data = text(kind, mb << 20)
        co = zlib.compressobj(6, zlib.DEFLATED, 31)
        want = co.compress(data) + co.flush()
        dev = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
        path = os.path.join(d, kind + ".gz")
        best_dev = best_host = 1e9
        for rep in range(3):
            torch.cuda.synchronize()
            t = time.perf_counter()
            with api.GpuGzWriter(path) as w:
                w.write(dev.data_ptr(), len(data), on_device=True)
            best_dev = min(best_dev, time.perf_counter() - t)
            assert open(path, "rb").read() == want, f"{kind}: GPU file differs from zlib"
            t = time.perf_counter()
            with api.GpuGzWriter(path) as w:
                w.write(data)
            best_host = min(best_host, time.perf_counter() - t)
            assert open(path, "rb").read() == want
        sample = data[:64 << 20]
        os.environ["PGB200_GZ"] = "host"
        t = time.perf_counter()
        with api.GpuGzWriter(path) as w:
            w.write(sample)
        t_zlib = time.perf_counter() - t
        del os.environ["PGB200_GZ"]
        res[kind] = {"bytes": len(data), "ratio": round(len(want) / len(data), 4),
                     "gpu_device_input_GBps": round(len(data) / best_dev / 1e9, 3),
                     "gpu_host_input_GBps": round(len(data) / best_host / 1e9, 3),
                     "zlib_gzwrite_MBps": round(len(sample) / t_zlib / 1e6, 1)}
    return res


def stage_numbers(a, d):
    import torch
    import bench
    from soapdenovo2_b200 import api
    ref_bin = os.path.join(ROOT, "oracle", "_ref", "SOAPdenovo-63mer")
    if not os.path.exists(ref_bin):
        raise SystemExit("oracle/_ref/SOAPdenovo-63mer is missing (it builds the map graph's contigs)")
    n_pairs = a.genome_len * a.coverage // 300
    t1, t2 = bench.gen_pe_fastq_gpu(torch, "cuda", a.genome_len, n_pairs, 42)
    t1.cpu().numpy().tofile(f"{d}/r_1.fq")
    t2.cpu().numpy().tofile(f"{d}/r_2.fq")
    del t1, t2
    torch.cuda.empty_cache()
    cfg = f"{d}/r.cfg"
    open(cfg, "w").write(f"max_rd_len=150\n[LIB]\navg_ins=300\nreverse_seq=0\nasm_flags=3\nrank=1\nq1={d}/r_1.fq\nq2={d}/r_2.fq\n")
    out = {}
    for mode in ("gpu", "host"):
        env = dict(os.environ, PGB200_GZ=mode, PGB200_VERBOSE="1")
        dt, _ = run([api.BIN63, "pregraph", "-s", cfg, "-K", str(a.K), "-p", "8", "-a", "16", "-R", "-o", f"{d}/pg_{mode}"], env)
        out[f"pregraph_wall_s_{mode}"] = round(dt, 2)
    for s in ("edge.gz", "vertex", "preArc", "preGraphBasic", "markOnEdge", "path"):
        if not filecmp.cmp(f"{d}/pg_gpu.{s}", f"{d}/pg_host.{s}", shallow=False):
            raise SystemExit(f"pregraph .{s} differs between PGB200_GZ=gpu and host")
    g = f"{d}/pg_gpu"
    run([ref_bin, "contig", "-g", g, "-R"], dict(os.environ))
    for mode in ("gpu", "host"):
        p = f"{d}/map_{mode}"
        for s in ("contig", "ContigIndex", "preGraphBasic"):
            shutil.copy(f"{g}.{s}", f"{p}.{s}")
        env = dict(os.environ, PGB200_GZ=mode, PGB200_VERBOSE="1")
        dt, err = run([api.BIN63, "map", "-s", cfg, "-g", p, "-p", "8"], env)
        out[f"map_wall_s_{mode}"] = round(dt, 2)
        m = re.search(r"record pass (\S+) ms, waiting for the deflate (\S+) ms", err)
        if m:
            out[f"map_record_pass_ms_{mode}"], out[f"map_deflate_wait_ms_{mode}"] = float(m.group(1)), float(m.group(2))
    for s in ("readOnContig.gz", "readInGap.gz", "peGrads"):
        if not filecmp.cmp(f"{d}/map_gpu.{s}", f"{d}/map_host.{s}", shallow=False):
            raise SystemExit(f"map .{s} differs between PGB200_GZ=gpu and host")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=int, default=512)
    ap.add_argument("--genome-len", type=int, default=100_000_000)
    ap.add_argument("--coverage", type=int, default=30)
    ap.add_argument("--K", type=int, default=63)
    ap.add_argument("--skip-stages", action="store_true")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", os.environ.get("PGB200_DEVICE", "0")],
                         capture_output=True, text=True).stdout.strip()
    d = tempfile.mkdtemp(prefix="pgb200_bench_gzip_")
    try:
        res = {"gpu": gpu, "writer": writer_numbers(a.mb, d)}
        if not a.skip_stages:
            res["stages"] = stage_numbers(a, d)
            res["stages"]["genome_len"], res["stages"]["coverage"] = a.genome_len, a.coverage
        print(json.dumps(res))
    finally:
        shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
