"""ctypes binding of libpregraph_b200.so (include/pregraph_b200.h) -- the Python-side mirror used by tests and bench.py.

The product is the C-ABI shared library + the `pregraph-b200-{63,127}mer` CLI; this module adds no compute of its own.
It fails loudly when the CUDA library has not been built: there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# PGB200_BUILD selects an alternative in-tree build directory pair lib_<name>/ bin_<name>/ (kernel tuning experiments: the same
# sources compiled with other -D parameters, `make -C soapdenovo2_b200/csrc VARIANT=<name> EXTRA=...`); default: lib/ and bin/.
_SFX = ("_" + os.environ["PGB200_BUILD"]) if os.environ.get("PGB200_BUILD") else ""
LIB_PATH = os.path.join(_HERE, "lib" + _SFX, "libpregraph_b200.so")
BIN63 = os.path.join(_HERE, "bin" + _SFX, "pregraph-b200-63mer")
BIN127 = os.path.join(_HERE, "bin" + _SFX, "pregraph-b200-127mer")

EXPORTS = [
    "pgb200_last_error", "pgb200_default_params", "pgb200_create", "pgb200_destroy", "pgb200_host_alloc", "pgb200_host_free",
    "pgb200_feed_text", "pgb200_last_chunk_records",
    "pgb200_xchg_setup", "pgb200_xchg_export", "pgb200_xchg_import", "pgb200_xchg_base", "pgb200_xchg_import_ptr", "pgb200_xchg_fence", "pgb200_flush", "pgb200_xchg_room", "pgb200_absorb",
    "pgb200_finish_pass1", "pgb200_reset_pass1", "pgb200_sweeps",
    "pgb200_build_layout", "pgb200_node_count", "pgb200_dump_nodes", "pgb200_sample_table", "pgb200_remove_tips", "pgb200_kmer2edges",
    "pgb200_read2edge", "pgb200_output_vertex", "pgb200_edge_text_to_sidecar", "pgb200_sidecar_to_edge_gz", "pgb200_plan_files", "pgb200_cut_chunk", "pgb200_pregraph_main", "pgb200_map_main", "call_pregraph",
]


class Params(C.Structure):
    _fields_ = [("K", C.c_int), ("P", C.c_int), ("initG", C.c_int), ("D", C.c_int), ("repsTie", C.c_int), ("flavour127", C.c_int),
                ("device", C.c_int), ("max_rd_len", C.c_int), ("table_slots", C.c_uint64), ("verbose", C.c_int), ("world", C.c_int),
                ("rank", C.c_int)]


class Pass1Stats(C.Structure):
    _fields_ = [("records", C.c_uint64), ("reads_kept", C.c_uint64), ("instances", C.c_uint64), ("distinct", C.c_uint64),
                ("table_slots", C.c_uint64), ("launches", C.c_uint64), ("ms_decode", C.c_double), ("ms_insert", C.c_double),
                ("ms_apply", C.c_double)]


class GraphStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("single_tips", "minor_tips", "num_ed", "edges", "extra_nodes", "deleted_reads", "arcs", "vertices")]


_lib = None


def load():
    """Load the shared library (raises if it was not built: the CUDA path is the only path)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` (no CPU fallback exists)")
    lib = C.CDLL(LIB_PATH)
    lib.pgb200_last_error.restype = C.c_char_p
    lib.pgb200_create.restype = C.c_void_p
    lib.pgb200_create.argtypes = [C.POINTER(Params)]
    lib.pgb200_destroy.argtypes = [C.c_void_p]
    lib.pgb200_host_alloc.restype = C.c_void_p
    lib.pgb200_host_alloc.argtypes = [C.c_size_t]
    lib.pgb200_host_free.argtypes = [C.c_void_p]
    lib.pgb200_feed_text.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_uint64, C.c_uint64, C.c_int, C.c_int]
    lib.pgb200_last_chunk_records.restype = C.c_uint64
    lib.pgb200_last_chunk_records.argtypes = [C.c_void_p]
    lib.pgb200_xchg_setup.argtypes = [C.c_void_p, C.c_uint64]
    lib.pgb200_xchg_export.argtypes = [C.c_void_p, C.c_void_p]
    lib.pgb200_xchg_import.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    lib.pgb200_xchg_base.restype = C.c_void_p
    lib.pgb200_xchg_base.argtypes = [C.c_void_p]
    lib.pgb200_xchg_import_ptr.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    lib.pgb200_xchg_fence.argtypes = [C.c_void_p]
    lib.pgb200_flush.argtypes = [C.c_void_p]
    lib.pgb200_xchg_room.argtypes = [C.c_void_p, C.c_uint64]
    lib.pgb200_absorb.argtypes = [C.c_void_p, C.c_void_p]
    lib.pgb200_finish_pass1.argtypes = [C.c_void_p, C.POINTER(Pass1Stats)]
    lib.pgb200_reset_pass1.argtypes = [C.c_void_p]
    lib.pgb200_sweeps.argtypes = [C.c_void_p, C.POINTER(C.c_longlong), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    lib.pgb200_build_layout.argtypes = [C.c_void_p]
    lib.pgb200_node_count.restype = C.c_uint64
    lib.pgb200_node_count.argtypes = [C.c_void_p]
    lib.pgb200_dump_nodes.argtypes = [C.c_void_p, C.c_void_p]
    lib.pgb200_sample_table.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    for fn in ("pgb200_remove_tips",):
        getattr(lib, fn).argtypes = [C.c_void_p, C.POINTER(GraphStats)]
    for fn in ("pgb200_kmer2edges", "pgb200_read2edge", "pgb200_output_vertex"):
        getattr(lib, fn).argtypes = [C.c_void_p, C.c_char_p, C.POINTER(GraphStats)]
    lib.pgb200_edge_text_to_sidecar.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_int, C.c_uint64, C.c_char_p]
    lib.pgb200_sidecar_to_edge_gz.argtypes = [C.c_char_p]
    lib.pgb200_plan_files.argtypes = [C.c_char_p, C.c_char_p, C.c_size_t]
    lib.pgb200_cut_chunk.restype = C.c_size_t
    lib.pgb200_cut_chunk.argtypes = [C.c_char_p, C.c_size_t, C.c_int]
    lib.pgb200_pregraph_main.argtypes = [C.c_int, C.POINTER(C.c_char_p), C.c_int]
    lib.pgb200_map_main.argtypes = [C.c_int, C.POINTER(C.c_char_p), C.c_int]
    _lib = lib
    return lib


class EngineError(RuntimeError):
    pass


class PregraphEngine:
    """One GPU's pregraph engine.  Method names follow the reference's phase functions (see include/pregraph_b200.h)."""

    def __init__(self, K=23, P=8, initG=0, D=0, repsTie=0, flavour127=0, device=0, max_rd_len=100, table_slots=0, verbose=0,
                 world=1, rank=0):
        self.lib = load()
        self.params = Params(K, P, initG, D, repsTie, flavour127, device, max_rd_len, table_slots, verbose, world, rank)
        self.h = self.lib.pgb200_create(C.byref(self.params))
        if not self.h:
            raise EngineError(self.lib.pgb200_last_error().decode())
        self.graph = GraphStats()

    def close(self):
        if self.h:
            self.lib.pgb200_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc:
            raise EngineError(self.lib.pgb200_last_error().decode())

    def feed_text(self, buf, nbytes=None, on_device=False, fastq=False, ord_base=0, ord_stride=1, reverse_seq=0, maxlen=None):
        """buf: bytes / bytearray / int address (host pinned or device pointer)."""
        if isinstance(buf, (bytes, bytearray)):
            n = len(buf) if nbytes is None else nbytes
            keep = (C.c_char * n).from_buffer_copy(buf) if isinstance(buf, bytes) else (C.c_char * n).from_buffer(buf)
            ptr = C.cast(keep, C.c_void_p)
        else:
            ptr, n = C.c_void_p(int(buf)), nbytes
        self._ck(self.lib.pgb200_feed_text(self.h, ptr, n, int(on_device), int(fastq), ord_base, ord_stride, reverse_seq,
                                           maxlen if maxlen is not None else self.params.max_rd_len))
        return self.lib.pgb200_last_chunk_records(self.h)

    # ---- multi-GPU record exchange (peer stores over NVLink): see include/pregraph_b200.h
    def xchg_setup(self, cap_records):
        self._ck(self.lib.pgb200_xchg_setup(self.h, cap_records))

    def xchg_export(self) -> bytes:
        h = C.create_string_buffer(64)
        self._ck(self.lib.pgb200_xchg_export(self.h, h))
        return h.raw

    def xchg_import(self, peer, handle: bytes):
        h = C.create_string_buffer(handle, 64)
        self._ck(self.lib.pgb200_xchg_import(self.h, peer, h))

    def xchg_base(self) -> int:
        return self.lib.pgb200_xchg_base(self.h) or 0

    def xchg_import_ptr(self, peer, peer_device, base):
        self._ck(self.lib.pgb200_xchg_import_ptr(self.h, peer, peer_device, C.c_void_p(int(base))))

    def xchg_fence(self):
        self._ck(self.lib.pgb200_xchg_fence(self.h))

    def flush(self):
        self._ck(self.lib.pgb200_flush(self.h))

    def xchg_room(self, n_rec) -> bool:
        return self.lib.pgb200_xchg_room(self.h, n_rec) == 1

    def absorb(self, other):
        self._ck(self.lib.pgb200_absorb(self.h, other.h))

    def finish_pass1(self) -> Pass1Stats:
        st = Pass1Stats()
        self._ck(self.lib.pgb200_finish_pass1(self.h, C.byref(st)))
        return st

    def reset_pass1(self):
        self._ck(self.lib.pgb200_reset_pass1(self.h))

    def sweeps(self):
        hist = (C.c_longlong * 256)()
        lin, rem = C.c_uint64(), C.c_uint64()
        self._ck(self.lib.pgb200_sweeps(self.h, hist, C.byref(lin), C.byref(rem)))
        return list(hist), lin.value, rem.value

    def build_layout(self):
        self._ck(self.lib.pgb200_build_layout(self.h))

    def dump_nodes(self) -> bytes:
        n = self.lib.pgb200_node_count(self.h)
        rec = (4 if self.params.flavour127 else 2) * 8 + 10
        buf = C.create_string_buffer(max(1, n * rec))
        self._ck(self.lib.pgb200_dump_nodes(self.h, buf))
        return buf.raw[: n * rec]

    def sample_table(self, seed, one_in, cap):
        """Seeded sample of the table (see pgb200_sample_table): a list of (key w0..w3, payload, rank) tuples sorted by key."""
        buf = (C.c_uint64 * (6 * max(1, cap)))()
        n = C.c_uint64()
        self._ck(self.lib.pgb200_sample_table(self.h, seed, one_in, buf, cap, C.byref(n)))
        if n.value > cap:
            raise EngineError(f"sample_table: {n.value} entries, more than cap={cap}")
        return sorted(tuple(buf[6 * i:6 * i + 6]) for i in range(n.value))

    def remove_tips(self):
        self._ck(self.lib.pgb200_remove_tips(self.h, C.byref(self.graph)))

    def kmer2edges(self, prefix):
        self._ck(self.lib.pgb200_kmer2edges(self.h, prefix.encode(), C.byref(self.graph)))

    def read2edge(self, prefix):
        self._ck(self.lib.pgb200_read2edge(self.h, prefix.encode(), C.byref(self.graph)))

    def output_vertex(self, prefix):
        self._ck(self.lib.pgb200_output_vertex(self.h, prefix.encode(), C.byref(self.graph)))


def plan_files(cfg: str):
    """Host logic only: [(mate, fastq, reverse_seq, cut, path)] in the order the reference opens the files, and max_rd_len."""
    lib = load()
    buf = C.create_string_buffer(1 << 20)
    if lib.pgb200_plan_files(cfg.encode(), buf, len(buf)):
        raise EngineError(lib.pgb200_last_error().decode())
    lines = buf.value.decode().splitlines()
    plan = []
    for l in lines[1:]:
        m, fq, rev, cut, path = l.split(" ", 4)
        plan.append((int(m), int(fq), int(rev), int(cut), path))
    return int(lines[0].split()[1]), plan


def cut_chunk(buf: bytes, fastq: bool) -> int:
    """Host logic only: offset at which the stage would cut this text buffer (0: it would read more first)."""
    return int(load().pgb200_cut_chunk(buf, len(buf), int(fastq)))


def kmerfreq_text(hist) -> bytes:
    """.kmerFreq = 255 lines, counts for coverage 1..255 (freqStat, prlHashReads.c:1104-1132)."""
    return "".join(f"{hist[i]}\n" for i in range(1, 256)).encode()


def edge_gz_to_sidecar(prefix: str, K: int, flavour127: int = 0):
    """Host only: `<prefix>.edge.gz` -> `<prefix>.edge.b200` (what the stage writes itself with PGB200_EDGE_SIDECAR=1)."""
    import gzip
    lib = load()
    text = gzip.open(prefix + ".edge.gz", "rb").read()
    num_ed = int(open(prefix + ".preGraphBasic").read().split("EDGEs")[1].split()[0])
    if lib.pgb200_edge_text_to_sidecar(text, len(text), K, flavour127, num_ed, (prefix + ".edge.b200").encode()):
        raise EngineError(lib.pgb200_last_error().decode())


def sidecar_to_edge_gz(prefix: str):
    """Host only: `<prefix>.edge.b200` -> the byte-identical `<prefix>.edge.gz`."""
    lib = load()
    if lib.pgb200_sidecar_to_edge_gz(prefix.encode()):
        raise EngineError(lib.pgb200_last_error().decode())
