"""ctypes mirror of include/mashgpu.h.

Names follow the reference's seams: Engine.sketch ~ sketchFile/sketchSequence jobs (Sketch.cpp:1147-1365),
Engine.dist ~ compare/compareSketches (CommandDistance.cpp:306-448), Engine.screen_* ~ hashSequence + reduce
(CommandScreen.cpp:484-599, 288-455).  Every call goes through libmashgpu.so; nothing here computes hashes,
merges or p-values on the host.
"""
import ctypes as C
import os

import numpy as np

ALPHABET_NUCLEOTIDE = "ACGT"                 # reference Sketch.h:25
ALPHABET_PROTEIN = "ACDEFGHIKLMNPQRSTVWY"    # reference Sketch.h:26

_HERE = os.path.dirname(os.path.abspath(__file__))

u64p = C.POINTER(C.c_uint64)
u32p = C.POINTER(C.c_uint32)
u8p = C.POINTER(C.c_uint8)
f64p = C.POINTER(C.c_double)


class MashGpuError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"mashgpu error {code}: {msg}")
        self.code = code


class SketchParams(C.Structure):
    """mashgpu_sketch_params (Sketch::Parameters subset, reference Sketch.h:34-109)."""
    _fields_ = [("kmer_size", C.c_int32), ("sketch_size", C.c_uint32), ("seed", C.c_uint32),
                ("use64", C.c_int32), ("noncanonical", C.c_int32), ("preserve_case", C.c_int32),
                ("alphabet", C.c_uint8 * 256), ("min_copies", C.c_uint32), ("target_cov", C.c_double),
                ("bloom_bytes", C.c_uint64)]

    @property
    def kmer_space(self):
        return float(sum(1 for a in self.alphabet if a)) ** self.kmer_size   # Sketch.cpp:509


class DistParams(C.Structure):
    """mashgpu_dist_params (arguments of compareSketches, reference CommandDistance.h:92)."""
    _fields_ = [("sketch_size", C.c_uint64), ("kmer_size", C.c_int32), ("kmer_space", C.c_double),
                ("max_distance", C.c_double), ("max_pvalue", C.c_double)]


class SketchSet(C.Structure):
    _fields_ = [("n", C.c_uint64), ("stride", C.c_uint64), ("hashes", C.c_void_p),
                ("n_hashes", C.c_void_p), ("length", C.c_void_p), ("on_device", C.c_int32)]


class Stats(C.Structure):
    _fields_ = [("kernel_launches", C.c_uint64), ("scan_kernel_ms", C.c_double), ("scan_kernel_launches", C.c_uint64),
                ("dist_kernel_ms", C.c_double), ("dist_kernel_launches", C.c_uint64), ("exact_reruns", C.c_uint64),
                ("translate_kernel_ms", C.c_double), ("translate_kernel_launches", C.c_uint64), ("taxonomy_ms", C.c_double),
                ("reads_events", C.c_uint64), ("reads_replay_ms", C.c_double), ("reads_peak_device_bytes", C.c_uint64),
                ("unit_stages", C.c_uint64), ("unit_peak_device_bytes", C.c_uint64)]


class TaxRow(C.Structure):
    """mashgpu_tax_row (one key of the reference's counts map, TaxCounts taxdb.hpp:40-46)."""
    _fields_ = [("taxid", C.c_uint64), ("tax_count", C.c_uint64), ("tax_hash_count", C.c_uint64),
                ("clade_count", C.c_uint64), ("clade_hash_count", C.c_uint64)]


TAX_NONE = 0xFFFFFFFF          # MASHGPU_TAX_NONE: a sketch without a taxID


def lib_path():
    return os.path.join(_HERE, "libmashgpu.so")


_lib = None


def load_library():
    """Load libmashgpu.so (built in-tree by __graft_entry__.build()). No fallback."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if not os.path.exists(path):
        raise ImportError(f"{path} is missing: build the CUDA extension first "
                          "(python -c 'import __graft_entry__ as g; g.build()'); there is no CPU fallback")
    L = C.CDLL(path)
    L.mashgpu_set_alphabet.restype = C.c_uint32
    L.mashgpu_set_alphabet.argtypes = [C.POINTER(SketchParams), C.c_char_p]
    L.mashgpu_device_count.restype = C.c_int
    L.mashgpu_create.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
    L.mashgpu_destroy.argtypes = [C.c_void_p]
    L.mashgpu_destroy.restype = None
    L.mashgpu_last_error.restype = C.c_char_p
    L.mashgpu_last_error.argtypes = [C.c_void_p]
    L.mashgpu_sketch_batch.argtypes = [C.c_void_p, C.POINTER(SketchParams), C.c_uint64, C.c_void_p, u64p, u32p, C.c_uint64,
                                       u64p, u32p, u32p, u64p]
    L.mashgpu_sketch_stream_dev.argtypes = [C.c_void_p, C.POINTER(SketchParams), C.c_void_p, u64p, C.c_uint64,
                                            C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.mashgpu_sketch_reads.argtypes = [C.c_void_p, C.POINTER(SketchParams), C.c_uint64, C.c_void_p, u64p, u64p, u32p, u32p, u64p]
    L.mashgpu_reads_open.argtypes = [C.c_void_p, C.POINTER(SketchParams), C.POINTER(C.c_void_p)]
    L.mashgpu_reads_feed.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, u64p, C.POINTER(C.c_int)]
    L.mashgpu_reads_finish.argtypes = [C.c_void_p, u64p, u32p, u32p, u64p]
    L.mashgpu_reads_close.argtypes = [C.c_void_p]
    L.mashgpu_unit_open.argtypes = [C.c_void_p, C.POINTER(SketchParams), C.POINTER(C.c_void_p)]
    L.mashgpu_unit_feed.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, u64p]
    L.mashgpu_unit_finish.argtypes = [C.c_void_p, u64p, u32p, u32p, u64p, u64p]
    L.mashgpu_unit_close.argtypes = [C.c_void_p]
    L.mashgpu_sketch_batch_packed.argtypes = [C.c_void_p, C.POINTER(SketchParams), u64p, C.c_uint64, u64p, C.c_uint64, u64p, C.c_uint64, u64p, u32p, u32p]
    L.mashgpu_host_pack.argtypes = [C.POINTER(SketchParams), C.c_uint64, C.c_void_p, u64p, C.c_int, u64p, u64p, C.c_uint64, u64p]
    L.mashgpu_hash_windows.argtypes = [C.c_void_p, C.POINTER(SketchParams), C.c_void_p, C.c_uint64, u64p, u8p]
    L.mashgpu_translate6.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_void_p]
    L.mashgpu_dist_open.argtypes = [C.c_void_p, C.POINTER(SketchSet), C.POINTER(SketchSet), C.POINTER(DistParams), C.POINTER(C.c_void_p)]
    L.mashgpu_dist_run.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, u32p, u32p, f64p, f64p, u8p]
    L.mashgpu_dist_run_dev.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.mashgpu_dist_run_list.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, u64p, u32p, u32p, f64p, f64p, u64p]
    L.mashgpu_dist_close.argtypes = [C.c_void_p]
    L.mashgpu_dist_set_prefilter.argtypes = [C.c_void_p, C.c_int]
    L.mashgpu_dist_set_triangle.argtypes = [C.c_void_p, C.c_int]
    L.mashgpu_dist_prefilter_stats.argtypes = [C.c_void_p, u64p, u64p, C.POINTER(C.c_int)]
    L.mashgpu_dist_pair_stats.argtypes = [C.c_void_p, u64p]
    L.mashgpu_dist_run_best.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint32, u32p, u32p, u32p, u32p, u32p, f64p, f64p]
    L.mashgpu_dist_run_best_dev.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.mashgpu_dist_set_best_capacity.argtypes = [C.c_void_p, C.c_uint64]
    L.mashgpu_dist_best_stats.argtypes = [C.c_void_p, u64p, u64p, u64p, f64p]
    L.mashgpu_dist_components.argtypes = [C.c_void_p, u32p, u64p]
    L.mashgpu_dist_components_dev.argtypes = [C.c_void_p, C.c_void_p, u64p, C.c_void_p]
    L.mashgpu_dist_spanning_forest.argtypes = [C.c_void_p, u32p, u32p, u32p, u32p, f64p, f64p, u64p, u64p]
    L.mashgpu_dist_spanning_forest_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                   u64p, u64p, C.c_void_p]
    L.mashgpu_dist_representatives.argtypes = [C.c_void_p, u32p, u32p, u32p, f64p, f64p, u64p, u64p]
    L.mashgpu_dist_representatives_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, u64p, u64p,
                                                   C.c_void_p]
    L.mashgpu_dist_set_representative_block.argtypes = [C.c_void_p, C.c_uint64]
    L.mashgpu_dist_neighbor_joining.argtypes = [C.c_void_p, u32p, f64p]
    L.mashgpu_neighbor_joining_matrix.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, u32p, f64p, C.c_void_p]
    L.mashgpu_dist_linkage.argtypes = [C.c_void_p, C.c_int, u32p, u32p, f64p, u32p, u64p]
    L.mashgpu_dist_linkage_cut.argtypes = [C.c_void_p, C.c_int, C.c_double, u32p, u32p, u32p, f64p, u32p, u64p, u64p, u64p]
    L.mashgpu_dist_set_linkage_cut_cta_max.argtypes = [C.c_void_p, C.c_uint64]
    L.mashgpu_dist_linkage_cut_stats.argtypes = [C.c_void_p, f64p]
    L.mashgpu_linkage_matrix.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_int, u32p, u32p, f64p, u32p, u64p, C.c_void_p]
    L.mashgpu_dist.argtypes = [C.c_void_p, C.POINTER(SketchSet), C.POINTER(SketchSet), C.POINTER(DistParams), u32p, u32p, f64p, f64p, u8p]
    L.mashgpu_within_open.argtypes = [C.c_void_p, C.POINTER(SketchSet), C.POINTER(SketchSet), C.c_double, C.POINTER(C.c_void_p)]
    L.mashgpu_within_run.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, u32p, u32p, f64p, f64p, u8p]
    L.mashgpu_within_run_dev.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p]
    L.mashgpu_within_close.argtypes = [C.c_void_p]
    L.mashgpu_screen_open.argtypes = [C.c_void_p, C.POINTER(SketchParams), C.POINTER(SketchSet), C.POINTER(C.c_void_p)]
    L.mashgpu_screen_feed.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    L.mashgpu_screen_feed_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    L.mashgpu_screen_finish.argtypes = [C.c_void_p, u64p, u64p, f64p, f64p, u64p, u64p, u32p]
    L.mashgpu_screen_counters.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), u64p]
    L.mashgpu_screen_merge_mixture.argtypes = [C.c_void_p, u64p, C.c_uint32]
    L.mashgpu_screen_close.argtypes = [C.c_void_p]
    L.mashgpu_screen_mixture_dev.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
    L.mashgpu_screen_merge_mixtures_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint64]
    L.mashgpu_screen_finish_hits.argtypes = [C.c_void_p, u32p, u64p, u64p, f64p, f64p, u64p, u64p]
    L.mashgpu_screen_reset.argtypes = [C.c_void_p]
    L.mashgpu_screen_hits_stats.argtypes = [C.c_void_p, u64p, u64p, f64p, f64p]
    L.mashgpu_dict_local_sort.argtypes = [C.c_void_p, C.POINTER(SketchSet), C.c_uint64, C.c_void_p, C.c_void_p, u64p, C.c_void_p]
    L.mashgpu_dict_split.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, u64p, C.c_uint32, u64p, C.c_void_p]
    L.mashgpu_dict_rank.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, u64p, C.c_void_p]
    L.mashgpu_dict_scatter.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, u64p, u64p, C.c_uint32, C.POINTER(SketchSet), C.c_uint64,
                                       C.c_void_p, C.c_void_p, C.c_void_p]
    L.mashgpu_dist_open_encoded.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64,
                                            C.POINTER(DistParams), C.POINTER(C.c_void_p)]
    L.mashgpu_screen_set_winner.argtypes = [C.c_void_p, C.c_int]
    L.mashgpu_taxonomy_open.argtypes = [C.c_void_p, C.c_uint64, u32p, u64p, C.POINTER(C.c_void_p)]
    L.mashgpu_taxonomy_close.argtypes = [C.c_void_p]
    L.mashgpu_screen_taxonomy.argtypes = [C.c_void_p, C.c_void_p, u32p, C.c_uint32, u64p, C.c_void_p, C.c_uint64, u64p, u64p, u64p, u64p, u8p]
    L.mashgpu_set_timing.argtypes = [C.c_void_p, C.c_int]
    L.mashgpu_get_stats.argtypes = [C.c_void_p, C.POINTER(Stats), C.c_int]
    _lib = L
    return L


def _p(a, t):
    return a.ctypes.data_as(t) if a is not None else None


LINKAGE_METHODS = {"average": 0, "complete": 1}


def _linkage_method(method):
    """a method name, or a raw integer passed through as is (the C ABI refuses unknown values)"""
    if isinstance(method, str):
        if method not in LINKAGE_METHODS:
            raise ValueError(f"linkage method must be one of {sorted(LINKAGE_METHODS)}, not {method!r}")
        return LINKAGE_METHODS[method]
    return int(method)


def _matrix_ld(d_matrix, n, ld):
    if not getattr(d_matrix, "is_cuda", False) or str(d_matrix.dtype) != "torch.float64":
        raise ValueError("d_matrix must be a CUDA float64 tensor")
    if ld is None:
        ld = d_matrix.stride(0) if d_matrix.dim() == 2 else n
    if n >= 1 and (n - 1) * ld + n > d_matrix.numel():
        raise ValueError(f"d_matrix holds {d_matrix.numel()} elements, fewer than an {n} x {n} matrix with ld {ld}")
    return int(ld)


def _linkage_outputs(n):
    m = max(int(n) - 1, 0)
    return {"id_lo": np.zeros(m, np.uint32), "id_hi": np.zeros(m, np.uint32), "height": np.zeros(m, np.float64),
            "size": np.zeros(m, np.uint32)}


def _linkage_pointers(out):
    return _p(out["id_lo"], u32p), _p(out["id_hi"], u32p), _p(out["height"], f64p), _p(out["size"], u32p)


def linkage_z(merges):
    """the (n - 1, 4) float64 Z of scipy.cluster.hierarchy from the merges of linkage() / linkage_matrix()"""
    return np.column_stack([merges["id_lo"].astype(np.float64), merges["id_hi"].astype(np.float64), merges["height"],
                            merges["size"].astype(np.float64)])


def _as_u8(s):
    if isinstance(s, (bytes, bytearray, memoryview)):
        return np.frombuffer(s, dtype=np.uint8)
    return np.ascontiguousarray(s, dtype=np.uint8)


class _Set:
    """Keeps the numpy arrays behind a mashgpu_sketch_set alive."""

    def __init__(self, hashes, n_hashes, length=None, on_device=False, n=None, stride=None):
        if on_device:
            self.c = SketchSet(n, stride, hashes, n_hashes, length, 1)
            return
        self.h = np.ascontiguousarray(hashes, np.uint64)
        if self.h.ndim != 2:
            raise ValueError("hashes must be (n, stride)")
        self.n = np.ascontiguousarray(n_hashes, np.uint32)
        self.l = np.ascontiguousarray(length if length is not None else np.ones(self.h.shape[0]), np.uint64)
        self.c = SketchSet(self.h.shape[0], self.h.shape[1], self.h.ctypes.data, self.n.ctypes.data, self.l.ctypes.data, 0)


class Engine:
    """One mashgpu context (one CUDA device)."""

    def __init__(self, device=0):
        self.lib = load_library()
        h = C.c_void_p()
        rc = self.lib.mashgpu_create(device, C.byref(h))
        if rc != 0:
            raise MashGpuError(rc, (self.lib.mashgpu_last_error(None) or b"").decode())
        self.h = h
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            self.lib.mashgpu_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise MashGpuError(rc, (self.lib.mashgpu_last_error(self.h) or b"").decode())

    # ---- parameters (sketchParameterSetup / setAlphabetFromString) --------------------------------------
    def params(self, k=21, s=1000, seed=42, alphabet=ALPHABET_NUCLEOTIDE, noncanonical=False, preserve_case=False, min_copies=1, target_cov=0.0,
               bloom_bytes=0):
        p = SketchParams()
        p.min_copies = min_copies
        p.target_cov = target_cov
        p.bloom_bytes = bloom_bytes
        p.kmer_size = k
        p.sketch_size = s
        p.seed = seed
        p.noncanonical = int(noncanonical)
        p.preserve_case = int(preserve_case)
        self.lib.mashgpu_set_alphabet(C.byref(p), alphabet.encode())
        return p

    # ---- hot path 1 ----------------------------------------------------------------------------------------
    def sketch(self, records, p, unit_of_record=None, n_units=None, counts=False):
        """records: list of byte strings / uint8 arrays.  Returns (hashes (n_units, s) u64, n u32, length u64[, counts])."""
        bufs = [_as_u8(r) for r in records]
        ptrs = (C.c_void_p * max(1, len(bufs)))(*[b.ctypes.data if b.size else None for b in bufs])
        lens = np.array([b.size for b in bufs], dtype=np.uint64)
        if unit_of_record is None:
            n_units = len(bufs)
            uor = None
        else:
            uor = np.ascontiguousarray(unit_of_record, np.uint32)
            if n_units is None:
                n_units = int(uor.max()) + 1 if uor.size else 0
        s = p.sketch_size
        out = np.zeros((n_units, s), np.uint64)
        out_n = np.zeros(n_units, np.uint32)
        out_len = np.zeros(n_units, np.uint64)
        out_c = np.zeros((n_units, s), np.uint32) if counts else None
        self._check(self.lib.mashgpu_sketch_batch(self.h, C.byref(p), len(bufs), C.cast(ptrs, C.c_void_p), _p(lens, u64p),
                                                  _p(uor, u32p), n_units, _p(out, u64p), _p(out_c, u32p), _p(out_n, u32p), _p(out_len, u64p)))
        return (out, out_n, out_len, out_c) if counts else (out, out_n, out_len)

    def sketch_reads(self, records, p, counts=False):
        """`mash sketch -r [-m] [-c]` of one read set.  Returns (hashes[:n], counts[:n] | None, records_used)."""
        bufs = [_as_u8(r) for r in records]
        ptrs = (C.c_void_p * max(1, len(bufs)))(*[b.ctypes.data if b.size else None for b in bufs])
        lens = np.array([b.size for b in bufs], dtype=np.uint64)
        s = p.sketch_size
        out = np.zeros(s, np.uint64); out_c = np.zeros(s, np.uint32) if counts else None
        n = C.c_uint32(0); used = C.c_uint64(0)
        self._check(self.lib.mashgpu_sketch_reads(self.h, C.byref(p), len(bufs), C.cast(ptrs, C.c_void_p), _p(lens, u64p), _p(out, u64p), _p(out_c, u32p),
                                                  C.byref(n), C.byref(used)))
        return out[:n.value].copy(), (out_c[:n.value].copy() if counts else None), used.value

    def reads_open(self, p):
        """A streaming `mash sketch -r` job: feed the read set in any number of pieces, then finish()."""
        return ReadsJob(self, p)

    def unit_open(self, p):
        """A streaming sketch unit (one unit of Engine.sketch, any size): feed its records in any number of pieces, then finish()."""
        return UnitJob(self, p)

    def host_pack(self, records, p, threads=1):
        """records -> (codes u64[ceil(L/32)], runs u64[n, 2], record_start u64[n_records + 1]) in the packed stream format
        (every record followed by one separator position).  No GPU involved."""
        bufs = [_as_u8(r) for r in records]
        ptrs = (C.c_void_p * max(1, len(bufs)))(*[b.ctypes.data if b.size else None for b in bufs])
        lens = np.array([b.size for b in bufs], dtype=np.uint64)
        total = int(lens.sum()) + len(bufs)
        codes = np.zeros(max(1, (total + 31) // 32), np.uint64)
        cap = 1 << 16
        while True:
            runs = np.zeros(2 * cap, np.uint64)
            n_runs = C.c_uint64(0)
            self._check(self.lib.mashgpu_host_pack(C.byref(p), len(bufs), C.cast(ptrs, C.c_void_p), _p(lens, u64p), threads, _p(codes, u64p),
                                                   _p(runs, u64p), cap, C.byref(n_runs)))
            if n_runs.value <= cap:
                break
            cap = int(n_runs.value)
        starts = np.zeros(len(bufs) + 1, np.uint64)
        starts[1:] = np.cumsum(lens + np.uint64(1))
        return codes, runs[:2 * n_runs.value].reshape(-1, 2).copy(), starts

    def sketch_packed(self, codes, stream_len, runs, unit_start, p, counts=False):
        """mashgpu_sketch_batch_packed: units of a caller-packed 2-bit stream.  Returns (hashes, n[, counts])."""
        codes = np.ascontiguousarray(codes, np.uint64); runs = np.ascontiguousarray(runs, np.uint64).reshape(-1)
        us = np.ascontiguousarray(unit_start, np.uint64)
        n_units = us.size - 1
        s = p.sketch_size
        out = np.zeros((n_units, s), np.uint64); out_n = np.zeros(n_units, np.uint32)
        out_c = np.zeros((n_units, s), np.uint32) if counts else None
        self._check(self.lib.mashgpu_sketch_batch_packed(self.h, C.byref(p), _p(codes, u64p), stream_len, _p(runs, u64p) if runs.size else None, runs.size // 2,
                                                         _p(us, u64p), n_units, _p(out, u64p), _p(out_c, u32p), _p(out_n, u32p)))
        return (out, out_n, out_c) if counts else (out, out_n)

    def sketch_stream_dev(self, p, d_stream_ptr, unit_start, d_out_hashes, d_out_n, d_out_counts=None, stream=None):
        us = np.ascontiguousarray(unit_start, np.uint64)
        self._check(self.lib.mashgpu_sketch_stream_dev(self.h, C.byref(p), d_stream_ptr, _p(us, u64p), us.size - 1,
                                                       d_out_hashes, d_out_counts, d_out_n, stream))

    def hash_windows(self, seq, p):
        b = _as_u8(seq)
        n = max(0, b.size - p.kmer_size + 1)
        h = np.zeros(max(1, n), np.uint64)
        v = np.zeros(max(1, n), np.uint8)
        self._check(self.lib.mashgpu_hash_windows(self.h, C.byref(p), b.ctypes.data, b.size, _p(h, u64p), _p(v, u8p)))
        return h[:n], v[:n].astype(bool)

    def translate6(self, d_seq_ptr, length, preserve_case, d_out_ptr):
        """Six-frame translation of `length` bases at device address d_seq_ptr into translated_length(length) bytes at
        d_out_ptr: the six peptides, each followed by a 0 byte, stops and unknown codons as 0."""
        self._check(self.lib.mashgpu_translate6(self.h, d_seq_ptr, length, int(preserve_case), d_out_ptr))

    # ---- hot path 2 ----------------------------------------------------------------------------------------
    def dist(self, ref, ref_n, ref_len, qry=None, qry_n=None, qry_len=None, *, sketch_size, k, kmer_space,
             max_distance=1.0, max_pvalue=1.0):
        """All pairs, query-major.  Returns a dict of (n_qry, n_ref) arrays: numer, denom, distance, pvalue, pass."""
        job = self.dist_open(ref, ref_n, ref_len, qry, qry_n, qry_len, sketch_size=sketch_size, k=k, kmer_space=kmer_space,
                             max_distance=max_distance, max_pvalue=max_pvalue)
        try:
            return job.run(0, job.n_qry)
        finally:
            job.close()

    def dist_open(self, ref, ref_n, ref_len, qry=None, qry_n=None, qry_len=None, *, sketch_size, k, kmer_space,
                  max_distance=1.0, max_pvalue=1.0):
        return DistJob(self, ref, ref_n, ref_len, qry, qry_n, qry_len, sketch_size, k, kmer_space, max_distance, max_pvalue)

    def within_open(self, ref, ref_n, qry=None, qry_n=None, *, max_error=0.05):
        """`mash within` job: containment of every query sketch in every reference sketch (qry None: the set against itself).
        max_error is compared as a double; the CLI's -e is a float, so pass float32(e) to reproduce it."""
        return WithinJob(self, ref, ref_n, qry, qry_n, max_error)

    def dist_open_encoded(self, d_rows, d_n_eff, d_length, n_rows, ref_begin, ref_count, *, sketch_size, k, kmer_space,
                          max_distance=1.0, max_pvalue=1.0, keepalive=None):
        """Job over dictionary-encoded rows in device memory (pointers); references = rows [ref_begin, ref_begin + ref_count)."""
        return DistJob.encoded(self, d_rows, d_n_eff, d_length, n_rows, ref_begin, ref_count, sketch_size, k, kmer_space,
                               max_distance, max_pvalue, keepalive)

    def neighbor_joining_matrix(self, d_matrix, n, ld=None, stream=None):
        """Neighbor-joining tree (DESIGN.md 3.10) of the n x n float64 matrix in the CUDA tensor d_matrix (row i at element i * ld;
        ld defaults to the row stride of a 2-D tensor, else n).  Only the lower triangle is read, and the whole matrix is overwritten.
        Returns {"parent": uint32[2n - 2], "length": float64[2n - 2]}: leaves 0..n-1, join s makes node n + s, the center 2n - 3 has
        parent 0xFFFFFFFF and length 0."""
        ld = _matrix_ld(d_matrix, n, ld)
        m = max(2 * int(n) - 2, 0)
        out = {"parent": np.zeros(m, np.uint32), "length": np.zeros(m, np.float64)}
        self._check(self.lib.mashgpu_neighbor_joining_matrix(self.h, d_matrix.data_ptr(), int(n), ld, _p(out["parent"], u32p),
                                                             _p(out["length"], f64p), stream))
        return out

    def linkage_matrix(self, d_matrix, n, ld=None, method="average", stream=None):
        """Average or complete linkage (DESIGN.md 3.11) of the n x n float64 matrix in the CUDA tensor d_matrix (row i at element
        i * ld; ld defaults to the row stride of a 2-D tensor, else n).  Only the lower triangle is read, and the first n columns of
        every row are overwritten.  Returns the n - 1 merges in merge order, scipy's Z layout: {"id_lo": uint32, "id_hi": uint32,
        "height": float64, "size": uint32, "rows_rescanned": int}; linkage_z() makes the (n - 1, 4) Z of it."""
        ld, out, rows = _matrix_ld(d_matrix, n, ld), _linkage_outputs(n), C.c_uint64(0)
        self._check(self.lib.mashgpu_linkage_matrix(self.h, d_matrix.data_ptr(), int(n), ld, _linkage_method(method),
                                                    *_linkage_pointers(out), C.byref(rows), stream))
        out["rows_rescanned"] = rows.value
        return out

    # ---- sharded dictionary build (device pointers; see mash_b200/shard.py) ----------------------------------
    def dict_local_sort(self, d_hashes, d_n_hashes, n, stride, sketch_size, d_keys, d_slots, stream=None):
        st = SketchSet(n, stride, d_hashes, d_n_hashes, None, 1)
        nv = C.c_uint64(0)
        self._check(self.lib.mashgpu_dict_local_sort(self.h, C.byref(st), sketch_size, d_keys, d_slots, C.byref(nv), stream))
        return nv.value

    def dict_split(self, d_keys, n, splitters, stream=None):
        spl = np.ascontiguousarray(splitters, np.uint64)
        counts = np.zeros(spl.size + 1, np.uint64)
        self._check(self.lib.mashgpu_dict_split(self.h, d_keys, n, _p(spl, u64p), spl.size + 1, _p(counts, u64p), stream))
        return [int(c) for c in counts]

    def dict_rank(self, d_keys, n, d_codes, stream=None):
        nd = C.c_uint64(0)
        self._check(self.lib.mashgpu_dict_rank(self.h, d_keys, n, d_codes, C.byref(nd), stream))
        return nd.value

    def dict_scatter(self, d_codes, d_slots, seg_counts, seg_base, d_n_hashes, n, stride, sketch_size, d_rows, d_n_eff, stream=None):
        sc = np.ascontiguousarray(seg_counts, np.uint64); sb = np.ascontiguousarray(seg_base, np.uint64)
        st = SketchSet(n, stride, 1, d_n_hashes, None, 1)          # the hashes themselves are not read again
        self._check(self.lib.mashgpu_dict_scatter(self.h, d_codes, d_slots, _p(sc, u64p), _p(sb, u64p), sc.size, C.byref(st), sketch_size,
                                                  d_rows, d_n_eff, stream))

    # ---- hot path 3 ----------------------------------------------------------------------------------------
    def screen_open(self, ref, ref_n, p, ref_len=None):
        return ScreenJob(self, ref, ref_n, p, ref_len)

    def taxonomy_open(self, parent, taxid):
        """Dense taxonomy in device memory: parent[i] = index of node i's parent (i for a root), taxid[i] its taxID."""
        return Taxonomy(self, parent, taxid)

    # ---- instrumentation -----------------------------------------------------------------------------------
    def set_timing(self, on=True):
        self._check(self.lib.mashgpu_set_timing(self.h, int(on)))

    def stats(self, reset=False):
        st = Stats()
        self._check(self.lib.mashgpu_get_stats(self.h, C.byref(st), int(reset)))
        return {f: getattr(st, f) for f, _ in Stats._fields_}


def _run_grid(job, fn, what, table, q_begin, q_count, outputs):
    """A host run of a pair grid: (q_count, n_ref) arrays of the named outputs of `table` ((name, dtype, pointer type) in the C
    argument order); the others are passed as NULL. `pass` comes back as bool."""
    unknown = set(outputs) - {name for name, _, _ in table}
    if unknown:
        raise ValueError(f"unknown {what} outputs {sorted(unknown)}")
    arrs = {name: np.zeros(q_count * job.n_ref, dt) for name, dt, _ in table if name in outputs}
    ptrs = [_p(arrs[name], pt) if name in arrs else None for name, _, pt in table]
    job.eng._check(fn(job.h, q_begin, q_count, *ptrs))
    out = {name: a.reshape(q_count, job.n_ref) for name, a in arrs.items()}
    if "pass" in out:
        out["pass"] = out["pass"].astype(bool)
    return out


class DistJob:
    def __init__(self, eng, ref, ref_n, ref_len, qry, qry_n, qry_len, sketch_size, k, kmer_space, max_distance, max_pvalue):
        self.eng = eng
        if isinstance(ref, _Set):
            self._ref = ref
            self._qry = qry
        else:
            self._ref = _Set(ref, ref_n, ref_len)
            self._qry = None if qry is None else _Set(qry, qry_n, qry_len)
        self.n_ref = int(self._ref.c.n)
        self.n_qry = self.n_ref if self._qry is None else int(self._qry.c.n)
        self.params = DistParams(sketch_size, k, kmer_space, max_distance, max_pvalue)
        h = C.c_void_p()
        eng._check(eng.lib.mashgpu_dist_open(eng.h, C.byref(self._ref.c), C.byref(self._qry.c) if self._qry is not None else None,
                                             C.byref(self.params), C.byref(h)))
        self.h = h

    @classmethod
    def encoded(cls, eng, d_rows, d_n_eff, d_length, n_rows, ref_begin, ref_count, sketch_size, k, kmer_space, max_distance, max_pvalue,
                keepalive=None):
        self = cls.__new__(cls)
        self.eng = eng
        self._ref = keepalive        # the caller's device arrays must outlive the job
        self._qry = None
        self.n_ref, self.n_qry = int(ref_count), int(n_rows)
        self.params = DistParams(sketch_size, k, kmer_space, max_distance, max_pvalue)
        h = C.c_void_p()
        eng._check(eng.lib.mashgpu_dist_open_encoded(eng.h, d_rows, d_n_eff, d_length, n_rows, ref_begin, ref_count, C.byref(self.params), C.byref(h)))
        self.h = h
        return self

    DIST_OUTPUTS = (("numer", np.uint32, u32p), ("denom", np.uint32, u32p), ("distance", np.float64, f64p), ("pvalue", np.float64, f64p),
                    ("pass", np.uint8, u8p))

    def run(self, q_begin, q_count, outputs=("numer", "denom", "distance", "pvalue", "pass")):
        """(q_count, n_ref) arrays of the named outputs; the others are passed as NULL (neither copied back nor allocated)."""
        return _run_grid(self, self.eng.lib.mashgpu_dist_run, "dist", self.DIST_OUTPUTS, q_begin, q_count, outputs)

    def run_list(self, q_begin, q_count, capacity):
        """Passing pairs only, sorted by pair index. Returns (n_pass, dict of arrays) -- arrays empty when n_pass > capacity."""
        idx = np.zeros(capacity, np.uint64); numer = np.zeros(capacity, np.uint32); denom = np.zeros(capacity, np.uint32)
        dist = np.zeros(capacity, np.float64); pv = np.zeros(capacity, np.float64); n = C.c_uint64(0)
        self.eng._check(self.eng.lib.mashgpu_dist_run_list(self.h, q_begin, q_count, capacity, _p(idx, u64p), _p(numer, u32p), _p(denom, u32p),
                                                           _p(dist, f64p), _p(pv, f64p), C.byref(n)))
        m = n.value if n.value <= capacity else 0
        return n.value, {"index": idx[:m], "numer": numer[:m], "denom": denom[:m], "distance": dist[:m], "pvalue": pv[:m]}

    def run_dev(self, q_begin, q_count, d_numer=None, d_denom=None, d_distance=None, d_pvalue=None, d_pass=None, stream=None):
        self.eng._check(self.eng.lib.mashgpu_dist_run_dev(self.h, q_begin, q_count, d_numer, d_denom, d_distance, d_pvalue, d_pass, stream))

    def run_best(self, q_begin, q_count, n_best):
        """The n_best nearest references of every query among its hits (pass and numer > 0), by (distance, reference index).
        Returns n_hits, n_total of shape (q_count,) and ref, numer, denom, distance, pvalue of shape (q_count, n_best) in rank
        order; entries past n_hits are zero."""
        shp = (q_count, max(0, min(int(n_best), 1024)))        # an n_best out of range is refused by the library
        n_hits = np.zeros(q_count, np.uint32); n_total = np.zeros(q_count, np.uint32)
        ref = np.zeros(shp, np.uint32); numer = np.zeros(shp, np.uint32); denom = np.zeros(shp, np.uint32)
        dist = np.zeros(shp, np.float64); pv = np.zeros(shp, np.float64)
        self.eng._check(self.eng.lib.mashgpu_dist_run_best(self.h, q_begin, q_count, n_best, _p(n_hits, u32p), _p(n_total, u32p), _p(ref, u32p),
                                                           _p(numer, u32p), _p(denom, u32p), _p(dist, f64p), _p(pv, f64p)))
        return {"n_hits": n_hits, "n_total": n_total, "ref": ref, "numer": numer, "denom": denom, "distance": dist, "pvalue": pv}

    def run_best_dev(self, q_begin, q_count, n_best, d_n_hits, d_n_total, d_ref, d_numer, d_denom, d_distance, d_pvalue, stream=None):
        self.eng._check(self.eng.lib.mashgpu_dist_run_best_dev(self.h, q_begin, q_count, n_best, d_n_hits, d_n_total, d_ref, d_numer, d_denom,
                                                               d_distance, d_pvalue, stream))

    def set_best_capacity(self, entries):
        """Candidate buffer of run_best in entries (0 = default); values below n_ref are raised to it."""
        self.eng._check(self.eng.lib.mashgpu_dist_set_best_capacity(self.h, int(entries)))

    def best_stats(self):
        blocks = C.c_uint64(0); splits = C.c_uint64(0); cands = C.c_uint64(0); ms = C.c_double(0)
        self.eng._check(self.eng.lib.mashgpu_dist_best_stats(self.h, C.byref(blocks), C.byref(splits), C.byref(cands), C.byref(ms)))
        return {"blocks_run": blocks.value, "blocks_split": splits.value, "candidates": cands.value, "select_ms": ms.value}

    def components(self):
        """Connected components of the hits (pass and numer > 0) of the lower triangle: (labels, n_edges), labels[i] = smallest
        query row of row i's component (np.uint32, n_qry entries).  Self and encoded jobs only."""
        labels = np.zeros(self.n_qry, np.uint32)
        n = C.c_uint64(0)
        self.eng._check(self.eng.lib.mashgpu_dist_components(self.h, _p(labels, u32p), C.byref(n)))
        return labels, n.value

    def components_dev(self, d_labels, stream=None):
        """components() into a device array of n_qry uint32; returns n_edges."""
        n = C.c_uint64(0)
        self.eng._check(self.eng.lib.mashgpu_dist_components_dev(self.h, d_labels, C.byref(n), stream))
        return n.value

    def spanning_forest(self):
        """Minimum spanning forest of the same graph as components(), under the order (distance, col, row): a dict of the edges in
        that order, row (> col), col, numer, denom, distance, pvalue (values as run() returns them for (q = row, r = col - ref_begin)),
        plus "rounds", the Boruvka rounds run.  Self and encoded jobs only."""
        m = max(self.n_qry - 1, 0)
        out = {"row": np.zeros(m, np.uint32), "col": np.zeros(m, np.uint32), "numer": np.zeros(m, np.uint32), "denom": np.zeros(m, np.uint32),
               "distance": np.zeros(m, np.float64), "pvalue": np.zeros(m, np.float64)}
        n, rounds = C.c_uint64(0), C.c_uint64(0)
        self.eng._check(self.eng.lib.mashgpu_dist_spanning_forest(self.h, _p(out["row"], u32p), _p(out["col"], u32p), _p(out["numer"], u32p),
                                                                  _p(out["denom"], u32p), _p(out["distance"], f64p), _p(out["pvalue"], f64p),
                                                                  C.byref(n), C.byref(rounds)))
        out = {k: v[:n.value] for k, v in out.items()}
        out["rounds"] = rounds.value
        return out

    def spanning_forest_dev(self, d_row, d_col, d_numer, d_denom, d_distance, d_pvalue, stream=None):
        """spanning_forest() into device arrays of n_qry - 1 entries (uint32 row, col, numer, denom; float64 distance, pvalue);
        returns (n_edges, n_rounds)."""
        n, rounds = C.c_uint64(0), C.c_uint64(0)
        self.eng._check(self.eng.lib.mashgpu_dist_spanning_forest_dev(self.h, d_row, d_col, d_numer, d_denom, d_distance, d_pvalue,
                                                                      C.byref(n), C.byref(rounds), stream))
        return n.value, rounds.value

    def representatives(self):
        """Greedy dereplication (DESIGN.md 3.12) of the graph of components(), in index order: sketch v is a representative iff no
        representative u < v has an edge {u, v}, and every other sketch goes to its adjacent representative of least (distance, smaller
        index, larger index).  A dict of rep (uint32, i itself for a representative), numer, denom, distance, pvalue (run()'s values for
        (q = max(i, rep), r = min(i, rep)), zeros for a representative), plus "n_reps" and "rounds".  Self jobs only."""
        n = self.n_qry
        out = {"rep": np.zeros(n, np.uint32), "numer": np.zeros(n, np.uint32), "denom": np.zeros(n, np.uint32),
               "distance": np.zeros(n, np.float64), "pvalue": np.zeros(n, np.float64)}
        reps, rounds = C.c_uint64(0), C.c_uint64(0)
        self.eng._check(self.eng.lib.mashgpu_dist_representatives(self.h, _p(out["rep"], u32p), _p(out["numer"], u32p), _p(out["denom"], u32p),
                                                                  _p(out["distance"], f64p), _p(out["pvalue"], f64p), C.byref(reps),
                                                                  C.byref(rounds)))
        out["n_reps"] = reps.value
        out["rounds"] = rounds.value
        return out

    def representatives_dev(self, d_rep, d_numer, d_denom, d_distance, d_pvalue, stream=None):
        """representatives() into device arrays of n_qry entries (uint32 rep, numer, denom; float64 distance, pvalue); returns
        (n_reps, rounds)."""
        reps, rounds = C.c_uint64(0), C.c_uint64(0)
        self.eng._check(self.eng.lib.mashgpu_dist_representatives_dev(self.h, d_rep, d_numer, d_denom, d_distance, d_pvalue, C.byref(reps),
                                                                      C.byref(rounds), stream))
        return reps.value, rounds.value

    def set_representative_block(self, rows):
        """Rows of one first-pass block of representatives() (0 = default, at most 32768); the result does not depend on it."""
        self.eng._check(self.eng.lib.mashgpu_dist_set_representative_block(self.h, int(rows)))

    def neighbor_joining(self):
        """Neighbor-joining tree (DESIGN.md 3.10) of every pair's distance of a self job, D(i, j) = run()'s distance at (q = i, r = j),
        j < i, whatever max_distance, max_pvalue and set_triangle say: {"parent": uint32[2n - 2], "length": float64[2n - 2]} as
        Engine.neighbor_joining_matrix returns them.  At least 3 sketches; encoded jobs are refused."""
        m = max(2 * self.n_qry - 2, 0)
        out = {"parent": np.zeros(m, np.uint32), "length": np.zeros(m, np.float64)}
        self.eng._check(self.eng.lib.mashgpu_dist_neighbor_joining(self.h, _p(out["parent"], u32p), _p(out["length"], f64p)))
        return out

    def linkage(self, method="average"):
        """Average or complete linkage (DESIGN.md 3.11) of every pair's distance of a self job, D(i, j) = run()'s distance at
        (q = i, r = j), j < i, whatever max_distance, max_pvalue and set_triangle say: the merges as Engine.linkage_matrix returns
        them.  At least 2 sketches; encoded jobs are refused."""
        out, rows = _linkage_outputs(self.n_qry), C.c_uint64(0)
        self.eng._check(self.eng.lib.mashgpu_dist_linkage(self.h, _linkage_method(method), *_linkage_pointers(out), C.byref(rows)))
        out["rows_rescanned"] = rows.value
        return out

    def linkage_cut(self, method, t, merges=False):
        """The flat clusters of linkage(method) cut at height t (DESIGN.md 3.13), linked per component of the pairs within about t, so
        the n x n matrix is never built: {"labels": uint32[n_qry], the smallest index of each sketch's cluster, "n_clusters",
        "n_components", "largest_component"}.  With merges=True also "merges", each component's own linkage in Z layout (leaves =
        sketch indices), n_qry - n_components entries grouped by component; those at height <= t are linkage()'s.  Self jobs only."""
        n = self.n_qry
        labels = np.zeros(n, np.uint32)
        out = _linkage_outputs(n) if merges else None
        ptrs = _linkage_pointers(out) if merges else (None, None, None, None)
        clusters, comps, largest = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        self.eng._check(self.eng.lib.mashgpu_dist_linkage_cut(self.h, _linkage_method(method), float(t), _p(labels, u32p), *ptrs, C.byref(clusters),
                                                              C.byref(comps), C.byref(largest)))
        res = {"labels": labels, "n_clusters": clusters.value, "n_components": comps.value, "largest_component": largest.value}
        if merges:
            res["merges"] = {k: v[:max(n - comps.value, 0)] for k, v in out.items()}
        return res

    def set_linkage_cut_cta_max(self, members):
        """The largest component linkage_cut() links inside one CTA (0 = default, the most that fits; 1 = every component through the
        matrix tier); the result does not depend on it."""
        self.eng._check(self.eng.lib.mashgpu_dist_set_linkage_cut_cta_max(self.h, int(members)))

    def linkage_cut_stats(self):
        """Device time in ms of the last linkage_cut()'s phases: components, grouping, cta, matrix."""
        ms = np.zeros(4, np.float64)
        self.eng._check(self.eng.lib.mashgpu_dist_linkage_cut_stats(self.h, _p(ms, f64p)))
        return dict(zip(("components", "grouping", "cta", "matrix"), ms.tolist()))

    def set_prefilter(self, mode):
        """-1 = auto (default), 0 = merge every pair, 1 = always probe the reference tiles first."""
        self.eng._check(self.eng.lib.mashgpu_dist_set_prefilter(self.h, int(mode)))

    def set_triangle(self, on=True):
        """Self comparison, lower triangle only (pairs with r >= q are not computed or written)."""
        self.eng._check(self.eng.lib.mashgpu_dist_set_triangle(self.h, int(on)))

    def prefilter_stats(self):
        probed = C.c_uint64(0); flagged = C.c_uint64(0); active = C.c_int(0)
        self.eng._check(self.eng.lib.mashgpu_dist_prefilter_stats(self.h, C.byref(probed), C.byref(flagged), C.byref(active)))
        pairs = C.c_uint64(0)
        self.eng._check(self.eng.lib.mashgpu_dist_pair_stats(self.h, C.byref(pairs)))
        return {"combos_probed": probed.value, "combos_flagged": flagged.value, "active": bool(active.value), "pairs_from_lists": pairs.value}

    def close(self):
        if self.h:
            self.eng.lib.mashgpu_dist_close(self.h)
            self.h = None


class WithinJob:
    def __init__(self, eng, ref, ref_n, qry, qry_n, max_error):
        self.eng = eng
        self._ref = ref if isinstance(ref, _Set) else _Set(ref, ref_n)
        self._qry = qry if (qry is None or isinstance(qry, _Set)) else _Set(qry, qry_n)
        self.n_ref = int(self._ref.c.n)
        self.n_qry = self.n_ref if self._qry is None else int(self._qry.c.n)
        h = C.c_void_p()
        eng._check(eng.lib.mashgpu_within_open(eng.h, C.byref(self._ref.c), C.byref(self._qry.c) if self._qry is not None else None,
                                               float(max_error), C.byref(h)))
        self.h = h

    WITHIN_OUTPUTS = (("common", np.uint32, u32p), ("examined", np.uint32, u32p), ("score", np.float64, f64p), ("error", np.float64, f64p),
                      ("pass", np.uint8, u8p))

    def run(self, q_begin, q_count, outputs=("common", "examined", "score", "error", "pass")):
        """(q_count, n_ref) arrays of the named outputs; the others are passed as NULL."""
        return _run_grid(self, self.eng.lib.mashgpu_within_run, "within", self.WITHIN_OUTPUTS, q_begin, q_count, outputs)

    def run_dev(self, q_begin, q_count, d_common=None, d_examined=None, d_score=None, d_error=None, d_pass=None, stream=None):
        self.eng._check(self.eng.lib.mashgpu_within_run_dev(self.h, q_begin, q_count, d_common, d_examined, d_score, d_error, d_pass, stream))

    def close(self):
        if self.h:
            self.eng.lib.mashgpu_within_close(self.h)
            self.h = None


class ReadsJob:
    def __init__(self, eng, p):
        self.eng = eng
        self.p = p
        h = C.c_void_p()
        eng._check(eng.lib.mashgpu_reads_open(eng.h, C.byref(p), C.byref(h)))
        self.h = h

    def feed(self, records):
        """The next records of the read set, in order.  Returns True once the target coverage (-c) was reached."""
        bufs = [_as_u8(r) for r in records]
        ptrs = (C.c_void_p * max(1, len(bufs)))(*[b.ctypes.data if b.size else None for b in bufs])
        lens = np.array([b.size for b in bufs], dtype=np.uint64)
        stopped = C.c_int(0)
        self.eng._check(self.eng.lib.mashgpu_reads_feed(self.h, len(bufs), C.cast(ptrs, C.c_void_p), _p(lens, u64p), C.byref(stopped)))
        return bool(stopped.value)

    def finish(self):
        """(hashes ascending, counts, records used) -- what Engine.sketch_reads returns with counts=True."""
        s = self.p.sketch_size
        out = np.zeros(s, np.uint64); out_c = np.zeros(s, np.uint32)
        n = C.c_uint32(0); used = C.c_uint64(0)
        self.eng._check(self.eng.lib.mashgpu_reads_finish(self.h, _p(out, u64p), _p(out_c, u32p), C.byref(n), C.byref(used)))
        return out[:n.value].copy(), out_c[:n.value].copy(), used.value

    def close(self):
        if self.h:
            self.eng.lib.mashgpu_reads_close(self.h)
            self.h = None


class UnitJob:
    def __init__(self, eng, p):
        self.eng = eng
        self.p = p
        h = C.c_void_p()
        eng._check(eng.lib.mashgpu_unit_open(eng.h, C.byref(p), C.byref(h)))
        self.h = h

    def feed(self, records):
        """The next records of the unit, in order."""
        bufs = [_as_u8(r) for r in records]
        ptrs = (C.c_void_p * max(1, len(bufs)))(*[b.ctypes.data if b.size else None for b in bufs])
        lens = np.array([b.size for b in bufs], dtype=np.uint64)
        self.eng._check(self.eng.lib.mashgpu_unit_feed(self.h, len(bufs), C.cast(ptrs, C.c_void_p), _p(lens, u64p)))

    def finish(self, counts=True):
        """(hashes ascending, counts | None, length, records): one row of Engine.sketch with the kept records' number."""
        s = self.p.sketch_size
        out = np.zeros(s, np.uint64); out_c = np.zeros(s, np.uint32) if counts else None
        n = C.c_uint32(0); length = C.c_uint64(0); recs = C.c_uint64(0)
        self.eng._check(self.eng.lib.mashgpu_unit_finish(self.h, _p(out, u64p), _p(out_c, u32p), C.byref(n), C.byref(length), C.byref(recs)))
        return out[:n.value].copy(), (out_c[:n.value].copy() if counts else None), length.value, recs.value

    def close(self):
        if self.h:
            self.eng.lib.mashgpu_unit_close(self.h)
            self.h = None


class ScreenJob:
    def __init__(self, eng, ref, ref_n, p, ref_len=None):
        self.eng = eng
        self._ref = ref if isinstance(ref, _Set) else _Set(ref, ref_n, ref_len)
        self.n_ref = int(self._ref.c.n)
        self.p = p
        h = C.c_void_p()
        eng._check(eng.lib.mashgpu_screen_open(eng.h, C.byref(p), C.byref(self._ref.c), C.byref(h)))
        self.h = h

    def feed(self, chunk):
        b = _as_u8(chunk)
        self.eng._check(self.eng.lib.mashgpu_screen_feed(self.h, b.ctypes.data, b.size))

    def feed_dev(self, d_ptr, length):
        self.eng._check(self.eng.lib.mashgpu_screen_feed_dev(self.h, d_ptr, length))

    def set_winner(self, on=True):
        """`mash screen -w`: reallocate every seen reference hash to the best sketch containing it before the reduce."""
        self.eng._check(self.eng.lib.mashgpu_screen_set_winner(self.h, int(on)))

    def counters(self):
        """(device pointer, slot count) of the uint32 hit counters, for an all-reduce across ranks."""
        ptr = C.c_void_p(); n = C.c_uint64(0)
        self.eng._check(self.eng.lib.mashgpu_screen_counters(self.h, C.byref(ptr), C.byref(n)))
        return ptr.value, n.value

    def merge_mixture(self, hashes):
        h = np.ascontiguousarray(hashes, np.uint64)
        self.eng._check(self.eng.lib.mashgpu_screen_merge_mixture(self.h, _p(h, u64p), h.size))

    def mixture_dev(self):
        """(device pointer of the running bottom-s list, device pointer of its length) for an all-gather across ranks."""
        a = C.c_void_p(); b = C.c_void_p()
        self.eng._check(self.eng.lib.mashgpu_screen_mixture_dev(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def merge_mixtures_dev(self, d_hashes, d_n, n_lists, stride):
        self.eng._check(self.eng.lib.mashgpu_screen_merge_mixtures_dev(self.h, d_hashes, d_n, n_lists, stride))

    def mixture(self):
        """The running bottom-s list of the mixture (ascending u64)."""
        return self.finish_mixture_only()

    def finish_mixture_only(self):
        s = self.p.sketch_size
        set_size = C.c_uint64(0); mix = np.zeros(s, np.uint64); mix_n = C.c_uint32(0)
        self.eng._check(self.eng.lib.mashgpu_screen_finish(self.h, None, None, None, None, C.byref(set_size), _p(mix, u64p), C.byref(mix_n)))
        return mix[:mix_n.value].copy()

    def finish(self):
        n, s = self.n_ref, self.p.sketch_size
        shared = np.zeros(n, np.uint64); median = np.zeros(n, np.uint64)
        ident = np.zeros(n, np.float64); pv = np.zeros(n, np.float64)
        set_size = C.c_uint64(0); mix = np.zeros(s, np.uint64); mix_n = C.c_uint32(0)
        self.eng._check(self.eng.lib.mashgpu_screen_finish(self.h, _p(shared, u64p), _p(median, u64p), _p(ident, f64p), _p(pv, f64p),
                                                           C.byref(set_size), _p(mix, u64p), C.byref(mix_n)))
        return dict(shared=shared, median=median, identity=ident, pvalue=pv, set_size=set_size.value, mixture=mix[:mix_n.value].copy())

    def finish_hits(self):
        """The sparse finish: finish()'s values at the references with shared >= 1 only, in ascending reference index.
        Returns dict(ref, shared, median, identity, pvalue (arrays of the rows), set_size)."""
        n = self.n_ref
        ref = np.zeros(max(1, n), np.uint32)
        shared = np.zeros(max(1, n), np.uint64); median = np.zeros(max(1, n), np.uint64)
        ident = np.zeros(max(1, n), np.float64); pv = np.zeros(max(1, n), np.float64)
        n_rows = C.c_uint64(0); set_size = C.c_uint64(0)
        self.eng._check(self.eng.lib.mashgpu_screen_finish_hits(self.h, _p(ref, u32p), _p(shared, u64p), _p(median, u64p), _p(ident, f64p),
                                                                _p(pv, f64p), C.byref(n_rows), C.byref(set_size)))
        m = n_rows.value
        return dict(ref=ref[:m].copy(), shared=shared[:m].copy(), median=median[:m].copy(), identity=ident[:m].copy(),
                    pvalue=pv[:m].copy(), set_size=set_size.value)

    def reset(self):
        """Start a new sample: hit counters and the mixture list emptied, the table kept."""
        self.eng._check(self.eng.lib.mashgpu_screen_reset(self.h))

    def hits_stats(self):
        """Of the last finish_hits(): dict(hit_hashes, hit_pairs, index_ms (the one-off index build), finish_ms)."""
        hh = C.c_uint64(0); hp = C.c_uint64(0); ims = C.c_double(0); fms = C.c_double(0)
        self.eng._check(self.eng.lib.mashgpu_screen_hits_stats(self.h, C.byref(hh), C.byref(hp), C.byref(ims), C.byref(fms)))
        return dict(hit_hashes=hh.value, hit_pairs=hp.value, index_ms=ims.value, finish_ms=fms.value)

    def taxonomy(self, tax, ref_code, unknown_taxid=(), hash_taxid=False):
        """`mash taxscreen` after the last feed: LCA taxon of every distinct hash, per-taxon counts and their roll-up.
        ref_code[r]: node index, n_nodes + u for unknown_taxid[u], or TAX_NONE.  Returns dict(rows (structured array of
        taxid, tax_count, tax_hash_count, clade_count, clade_hash_count), total_count, total_hash_count,
        hash_taxid (ascending hash order, or None), unknown_in_lca)."""
        code = np.ascontiguousarray(ref_code, np.uint32)
        unk = np.ascontiguousarray(unknown_taxid, np.uint64)
        cap = tax.n_nodes + unk.size + 2
        rows = (TaxRow * cap)()
        n_rows = C.c_uint64(0); tc = C.c_uint64(0); thc = C.c_uint64(0)
        _, n_distinct = self.counters()
        ht = np.zeros(max(1, n_distinct), np.uint64) if hash_taxid else None
        flags = np.zeros(max(1, unk.size), np.uint8)
        self.eng._check(self.eng.lib.mashgpu_screen_taxonomy(self.h, tax.h, _p(code, u32p) if code.size else None, unk.size,
                                                             _p(unk, u64p) if unk.size else None, C.cast(rows, C.c_void_p), cap,
                                                             C.byref(n_rows), C.byref(tc), C.byref(thc), _p(ht, u64p), _p(flags, u8p)))
        out = np.frombuffer(rows, dtype=np.dtype([(f, "<u8") for f, _ in TaxRow._fields_]))[:n_rows.value].copy()
        return dict(rows=out, total_count=tc.value, total_hash_count=thc.value,
                    hash_taxid=ht[:n_distinct].copy() if hash_taxid else None, unknown_in_lca=flags[:unk.size].astype(bool))

    def close(self):
        if self.h:
            self.eng.lib.mashgpu_screen_close(self.h)
            self.h = None


class Taxonomy:
    def __init__(self, eng, parent, taxid):
        self.eng = eng
        self.parent = np.ascontiguousarray(parent, np.uint32)
        self.taxid = np.ascontiguousarray(taxid, np.uint64)
        self.n_nodes = int(self.taxid.size)
        h = C.c_void_p()
        eng._check(eng.lib.mashgpu_taxonomy_open(eng.h, self.n_nodes, _p(self.parent, u32p), _p(self.taxid, u64p), C.byref(h)))
        self.h = h

    def close(self):
        if self.h:
            self.eng.lib.mashgpu_taxonomy_close(self.h)
            self.h = None
