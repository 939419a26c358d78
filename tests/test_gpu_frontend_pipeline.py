"""The pass-1 front end under chunk patterns the parity suite does not feed: dozens of chunks of very unequal size (so every per-chunk
buffer is reused by small and large chunks alternately), aggregation launches between them, reads with more runs than a side row
holds in consecutive chunks, and a second pass that starts while the table clear queued by reset_pass1 is still running.  Every case
must give the oracle's node table bit for bit."""
import itertools

import pytest

from soapdenovo2_b200 import api, synth
from tests import util

pytestmark = pytest.mark.gpu

CHUNK_READS = (1, 2, 700, 1, 3000, 5, 64, 1, 1200)   # unequal: a buffer sized by a large chunk is reused by a chunk of one read


@pytest.fixture(scope="module", autouse=True)
def _build():
    util.build_oracle()


def _records(path, fastq):
    lines = open(path, "rb").read().split(b"\n")[:-1]
    lpr = 4 if fastq else 2
    return [b"\n".join(lines[i:i + lpr]) + b"\n" for i in range(0, len(lines), lpr)]


def _feed_in_chunks(eng, recs, fastq, sizes, mate=None):
    """Feeds recs in chunks of the given sizes (cycled); mate None: single-end ordinals, else the ordinals of that mate of a pair."""
    i = 0
    for n in itertools.cycle(sizes):
        if i >= len(recs):
            break
        part = recs[i:i + n]
        if mate is None:
            eng.feed_text(b"".join(part), fastq=fastq, ord_base=i)
        else:
            eng.feed_text(b"".join(part), fastq=fastq, ord_base=2 * i + mate, ord_stride=2)
        i += len(part)


def _check_table(eng, mod, dump):
    eng.finish_pass1()
    hist, _, _ = eng.sweeps()
    assert api.kmerfreq_text(hist) == open(mod + ".kmerFreq", "rb").read()
    eng.build_layout()
    assert eng.dump_nodes() == open(dump, "rb").read()


@pytest.mark.parametrize("stress", [False, True], ids=["plain", "arena1mb_flush2"])
@pytest.mark.parametrize("kind,K", [("pe_fastq", 63), ("se_fasta", 31), ("pe_fastq", 127)])
def test_unequal_chunks(tmp_path, monkeypatch, kind, K, stress):
    """Dozens of chunks of 1 .. 3000 reads; with a 1 MB arena and an aggregation every second chunk, aggregation launches land between
    the chunks' partitions and the table grows from 2048 slots."""
    monkeypatch.setenv("PGB200_SKM", "1")
    if stress:
        monkeypatch.setenv("PGB200_SKM_ARENA_MB", "1")
        monkeypatch.setenv("PGB200_SKM_FLUSH_EVERY", "2")
    sizes = tuple(min(n, 800) for n in CHUNK_READS) if stress else CHUNK_READS   # a chunk's records must fit the 1 MB arena
    flav = int(K > 63)
    mod, dump = str(tmp_path / "mod"), str(tmp_path / "mod.table")
    if kind == "pe_fastq":
        cfg = synth.scenario_pe_fastq(str(tmp_path))
        util.run_model(util.MODEL127 if flav else util.MODEL63, cfg, mod, K, 4, ("-1", "-T", dump, "-a", "1"))
        eng = api.PregraphEngine(K=K, P=4, initG=1, flavour127=flav, max_rd_len=150, table_slots=2048 if stress else 0)
        for mate, fn in enumerate(("pe_1.fq", "pe_2.fq")):
            _feed_in_chunks(eng, _records(tmp_path / fn, True), True, sizes, mate)
    else:
        cfg = synth.scenario_se_fasta(str(tmp_path), n_reads=9000)
        util.run_model(util.MODEL63, cfg, mod, K, 4, ("-1", "-T", dump, "-a", "1"))
        eng = api.PregraphEngine(K=K, P=4, initG=1, max_rd_len=100, table_slots=2048 if stress else 0)
        _feed_in_chunks(eng, _records(tmp_path / "se.fa", False), False, sizes)
    _check_table(eng, mod, dump)
    eng.close()


def test_reads_with_many_runs_in_consecutive_chunks(tmp_path, monkeypatch):
    """800-base reads at K = 31: a run is at most K - m + 1 <= 31 k-mers long, so the 770 k-mers of a read make more than the 16 runs
    a side row holds and the read goes through k_skm_rescan, which reads the run counts its own chunk's count wrote.  Chunks of 1, 2, 1, 40
    reads put such reads into consecutive chunks that reuse the same side buffer."""
    monkeypatch.setenv("PGB200_SKM", "1")
    cfg = synth.scenario_se_fasta(str(tmp_path), genome_len=20000, n_reads=300, rd_len=800)
    mod, dump = str(tmp_path / "mod"), str(tmp_path / "mod.table")
    util.run_model(util.MODEL63, cfg, mod, 31, 3, ("-1", "-T", dump, "-a", "1"))
    eng = api.PregraphEngine(K=31, P=3, initG=1, max_rd_len=800)
    _feed_in_chunks(eng, _records(tmp_path / "se.fa", False), False, (1, 2, 1, 40))
    _check_table(eng, mod, dump)
    eng.close()


@pytest.mark.parametrize("mode", ["direct", "aggregated"])
def test_second_pass_joins_the_table_clear(tmp_path, monkeypatch, mode):
    """Two passes on one engine whose table (2^27 slots, 4.3 GB) takes far longer to clear than the small input takes to decode and
    partition: the second pass's first table access must wait for the clear that reset_pass1 queued, so it gives the first pass's
    table."""
    monkeypatch.setenv("PGB200_SKM", "0" if mode == "direct" else "1")
    cfg = synth.scenario_pe_fastq(str(tmp_path))
    mod, dump = str(tmp_path / "mod"), str(tmp_path / "mod.table")
    util.run_model(util.MODEL63, cfg, mod, 63, 4, ("-1", "-T", dump, "-a", "1"))
    eng = api.PregraphEngine(K=63, P=4, initG=1, max_rd_len=150, table_slots=1 << 27)
    for _ in range(3):
        for mate, fn in enumerate(("pe_1.fq", "pe_2.fq")):
            _feed_in_chunks(eng, _records(tmp_path / fn, True), True, (3000, 1, 1200), mate)
        _check_table(eng, mod, dump)
        eng.reset_pass1()
    eng.close()


@pytest.mark.parametrize("K,flav,D,buckets", [(63, 0, 2, "2"), (31, 0, 1, "3"), (127, 1, 2, "2")])
def test_fused_sweeps_when_a_key_is_both_spilled_and_claimed(tmp_path, monkeypatch, K, flav, D, buckets):
    """Two or three buckets: every bucket overflows its shared-memory table, so thousands of lanes meet the table's claim limit, and
    some key is spilled to the global table by one lane while another lane claims it in shared memory.  The flush merges such a key
    unswept and the spill list sweeps it, with -d too (a swept partial aggregate would have lost its low link counters for good).
    Three passes, each equal to the oracle."""
    monkeypatch.setenv("PGB200_SKM", "1")
    monkeypatch.setenv("PGB200_SKM_BUCKETS", buckets)
    cfg = synth.scenario_pe_fastq(str(tmp_path))
    mod, dump = str(tmp_path / "mod"), str(tmp_path / "mod.table")
    util.run_model(util.MODEL127 if flav else util.MODEL63, cfg, mod, K, 4, ("-1", "-T", dump, "-a", "1", "-d", str(D)))
    eng = api.PregraphEngine(K=K, P=4, initG=1, D=D, flavour127=flav, max_rd_len=150)
    for _ in range(3):
        for mate, fn in enumerate(("pe_1.fq", "pe_2.fq")):
            eng.feed_text(open(tmp_path / fn, "rb").read(), fastq=True, ord_base=mate, ord_stride=2)
        _check_table(eng, mod, dump)
        eng.reset_pass1()
    eng.close()
