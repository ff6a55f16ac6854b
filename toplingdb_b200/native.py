"""ctypes binding of include/b200c.h.  Fails loudly when the CUDA library is missing: there is no CPU path."""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B200C_LIB") or os.path.join(HERE, "libb200c.so")  # B200C_LIB: debugging override

OK, ERR_INVALID_ARGUMENT, ERR_NO_DEVICE, ERR_CUDA, ERR_CORRUPTION, ERR_NOT_SUPPORTED, ERR_OOM, ERR_STATE = range(8)
MEM_HOST, MEM_DEVICE, MEM_HOST_DEFERRED = 0, 1, 2
CKSUM = {"none": 0, "crc32c": 1, "xxh3": 4}
DBG_DECODED_KEYS, DBG_DECODED_VALUES, DBG_MERGED_KEYS, DBG_MERGED_VALUES, DBG_BLOCK_LIST = 1, 2, 3, 4, 5


class B200cError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"b200c error {code}: {msg}")
        self.code = code


class Grandparent(C.Structure):
    _fields_ = [("smallest_user_key", C.c_char_p), ("smallest_len", C.c_uint32), ("largest_user_key", C.c_char_p),
                ("largest_len", C.c_uint32), ("file_size", C.c_uint64)]


class Params(C.Structure):
    _fields_ = [
        ("abi_version", C.c_uint32), ("device", C.c_int32), ("output_level", C.c_int32), ("bottommost_level", C.c_int32),
        ("max_output_file_size", C.c_uint64), ("block_size", C.c_uint32), ("block_size_deviation", C.c_uint32),
        ("block_restart_interval", C.c_uint32), ("index_block_restart_interval", C.c_uint32), ("format_version", C.c_uint32),
        ("checksum", C.c_uint32), ("verify_input_checksums", C.c_uint32), ("snapshots", C.POINTER(C.c_uint64)),
        ("num_snapshots", C.c_uint32), ("column_family_id", C.c_uint32), ("column_family_name", C.c_char_p),
        ("db_id", C.c_char_p), ("db_session_id", C.c_char_p), ("db_host_id", C.c_char_p), ("creation_time", C.c_uint64),
        ("oldest_key_time", C.c_uint64), ("file_creation_times", C.POINTER(C.c_uint64)),
        ("num_file_creation_times", C.c_uint32), ("first_file_number", C.c_uint64), ("output_mem", C.c_uint32),
        ("profile", C.c_uint32), ("compaction_filter", C.c_uint32), ("ttl", C.c_int32), ("ttl_now", C.c_int64),
        ("grandparents", C.POINTER(Grandparent)), ("num_grandparents", C.c_uint32),
        ("level_compaction_dynamic_file_size", C.c_uint32), ("max_compaction_bytes", C.c_uint64),
        ("target_output_file_size", C.c_uint64),
        ("range_start_user_key", C.c_char_p), ("range_start_len", C.c_uint32), ("has_range_start", C.c_uint32),
        ("range_end_user_key", C.c_char_p), ("range_end_len", C.c_uint32), ("has_range_end", C.c_uint32),
        ("paranoid_file_checks", C.c_uint32), ("bloom_millibits_per_key", C.c_uint32),
        ("earliest_write_conflict_snapshot", C.c_uint64), ("sst_partitioner_prefix_len", C.c_uint32),
    ]


class FileMeta(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("file_number", "file_size", "smallest_seqno", "largest_seqno", "num_entries",
                                          "num_deletions", "raw_key_size", "raw_value_size", "num_data_blocks", "data_size",
                                          "index_size")] + [
        ("smallest_ikey_len", C.c_uint32), ("largest_ikey_len", C.c_uint32), ("smallest_ikey", C.c_uint8 * 64),
        ("largest_ikey", C.c_uint8 * 64)]


class JobStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("num_input_records", "num_output_records", "num_input_deletion_records",
                                          "num_records_replaced", "num_expired_deletion_records",
                                          "total_input_raw_key_bytes", "total_input_raw_value_bytes", "total_input_bytes",
                                          "total_output_bytes", "num_input_files", "num_output_files")] + [
        ("decode_us", C.c_double), ("merge_us", C.c_double), ("encode_us", C.c_double), ("total_us", C.c_double),
        ("kernel_launches", C.c_uint64), ("num_record_drop_user", C.c_uint64)]


_lib = None

EXPORTS = ["b200c_last_error", "b200c_abi_version", "b200c_device_count", "b200c_params_init", "b200c_job_create",
           "b200c_job_add_input", "b200c_job_run", "b200c_job_output_count", "b200c_job_output_meta",
           "b200c_job_output_data", "b200c_job_output_read", "b200c_job_get_stats", "b200c_job_destroy",
           "b200c_job_run_until", "b200c_job_debug_read", "b200c_block_checksums", "b200c_job_kernel_time_count",
           "b200c_job_kernel_time", "b200c_job_encode_columns", "b200c_host_alloc", "b200c_host_free", "b200c_job_encode_kv",
           "b200c_job_plan_ranges", "b200c_job_create_sub", "b200c_job_upload_by_ranges"]


def load_library(build_if_missing=True):
    """Loads libb200c.so; raises if it cannot be built/loaded (no silent fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        if not build_if_missing:
            raise B200cError(ERR_STATE, f"{LIB_PATH} is missing: run `python -m toplingdb_b200.build`")
        from . import build
        build.build_native()
    L = C.CDLL(LIB_PATH)
    L.b200c_last_error.restype = C.c_char_p
    L.b200c_abi_version.restype = C.c_uint32
    L.b200c_job_create.argtypes = [C.POINTER(Params), C.POINTER(C.c_void_p)]
    L.b200c_job_add_input.argtypes = [C.c_void_p, C.c_int, C.c_uint64, C.c_void_p, C.c_uint64, C.c_int]
    L.b200c_job_run.argtypes = [C.c_void_p]
    L.b200c_job_run_until.argtypes = [C.c_void_p, C.c_int]
    L.b200c_job_output_count.argtypes = [C.c_void_p]
    L.b200c_job_output_meta.argtypes = [C.c_void_p, C.c_int, C.POINTER(FileMeta)]
    L.b200c_job_output_data.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]
    L.b200c_job_output_read.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_uint64]
    L.b200c_job_get_stats.argtypes = [C.c_void_p, C.POINTER(JobStats)]
    L.b200c_job_destroy.argtypes = [C.c_void_p]
    L.b200c_job_destroy.restype = None
    L.b200c_job_debug_read.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    L.b200c_block_checksums.argtypes = [C.c_int, C.c_uint32, C.c_char_p, C.POINTER(C.c_uint64), C.c_uint32, C.c_uint8,
                                        C.POINTER(C.c_uint32)]
    L.b200c_job_kernel_time_count.argtypes = [C.c_void_p]
    L.b200c_job_kernel_time.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_double)]
    L.b200c_job_encode_columns.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.b200c_job_encode_kv.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]
    L.b200c_params_init.argtypes = [C.POINTER(Params)]
    L.b200c_params_init.restype = None
    L.b200c_job_plan_ranges.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64, C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    L.b200c_job_create_sub.argtypes = [C.c_void_p, C.POINTER(Params), C.POINTER(C.c_void_p)]
    L.b200c_job_upload_by_ranges.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32), C.c_uint32]
    _lib = L
    return L


def lib():
    return load_library()


def _check(rc):
    if rc != 0:
        raise B200cError(rc, lib().b200c_last_error().decode(errors="replace"))


def device_count():
    return lib().b200c_device_count()


def block_checksums(kind, buffers, last_byte=0, device=0):
    """Block checksum (table/format.cc:468-509) of each buffer, computed by the device kernels."""
    L = lib()
    offs = [0]
    for b in buffers:
        offs.append(offs[-1] + len(b))
    data = b"".join(buffers) + b"\0"
    out = (C.c_uint32 * max(1, len(buffers)))()
    _check(L.b200c_block_checksums(device, CKSUM[kind], data, (C.c_uint64 * len(offs))(*offs), len(buffers), last_byte, out))
    return list(out)[: len(buffers)]


class CompactionJob:
    """One compaction job = what CompactionExecutor::Execute receives (db/compaction/compaction_executor.h:160-178).

    Keyword arguments are the b200c_params fields; `checksum` takes "xxh3" / "crc32c" / "none".  `sst_partitioner_prefix_len=N`
    cuts the output files where the first N bytes of the user key change (SstPartitionerFixedPrefixFactory(N); 0 = none)."""

    def __init__(self, parent=None, **kw):
        L = lib()
        p = Params()
        L.b200c_params_init(C.byref(p))
        self._keep = []
        self._kw = dict(kw)
        for k, v in kw.items():
            if k == "checksum":
                p.checksum = CKSUM[v]
            elif k == "snapshots":
                arr = (C.c_uint64 * max(1, len(v)))(*v)
                self._keep.append(arr)
                p.snapshots = C.cast(arr, C.POINTER(C.c_uint64))
                p.num_snapshots = len(v)
            elif k == "file_creation_times":
                arr = (C.c_uint64 * max(1, len(v)))(*v)
                self._keep.append(arr)
                p.file_creation_times = C.cast(arr, C.POINTER(C.c_uint64))
                p.num_file_creation_times = len(v)
            elif k in ("column_family_name", "db_id", "db_session_id", "db_host_id"):
                b = v.encode() if isinstance(v, str) else v
                self._keep.append(b)
                setattr(p, k, b)
            elif k == "output_mem":
                p.output_mem = {"host": MEM_HOST, "device": MEM_DEVICE}.get(v, v)
            elif k == "bottommost_level":
                p.bottommost_level = int(v)
            elif k == "grandparents":  # [(smallest user key, largest user key, file size)]
                arr = (Grandparent * max(1, len(v)))()
                for i, (a, b, sz) in enumerate(v):
                    arr[i].smallest_user_key, arr[i].smallest_len = a, len(a)
                    arr[i].largest_user_key, arr[i].largest_len = b, len(b)
                    arr[i].file_size = sz
                    self._keep += [a, b]
                self._keep.append(arr)
                p.grandparents = C.cast(arr, C.POINTER(Grandparent))
                p.num_grandparents = len(v)
            elif k in ("range_start", "range_end"):  # sub-compaction key range: start <= user key < end; None = unbounded
                if v is not None:
                    v = bytes(v)
                    self._keep.append(v)
                    setattr(p, k + "_user_key", v)
                    setattr(p, k + "_len", len(v))
                    setattr(p, "has_" + k, 1)
            elif k == "compaction_filter":
                p.compaction_filter = {"none": 0, "remove_empty_value": 1, "ttl": 2}.get(v, v)
            else:
                if not hasattr(p, k):
                    raise TypeError(f"unknown job parameter {k}")
                setattr(p, k, v)
        self.params = p
        self._h = C.c_void_p()
        self._parent = parent  # a sub-job keeps its parent (and with it the shared input images) alive
        if parent is not None:
            parent._wait_for_torch()
            _check(L.b200c_job_create_sub(parent._h, C.byref(p), C.byref(self._h)))
        else:
            _check(L.b200c_job_create(C.byref(p), C.byref(self._h)))
        self.ninputs = parent.ninputs if parent is not None else 0
        self._torch_device_inputs = False

    def plan_ranges(self, max_ranges, min_range_bytes=0):
        """boundary user keys of up to max_ranges key ranges of about equal input bytes (GenSubcompactionBoundaries' job)"""
        n = max(1, max_ranges)
        keys = C.create_string_buffer(16 * n)
        lens = (C.c_uint32 * n)()
        nb = C.c_uint32()
        self._wait_for_torch()
        _check(lib().b200c_job_plan_ranges(self._h, max_ranges, min_range_bytes, keys, lens, C.byref(nb)))
        return [keys.raw[16 * i:16 * i + lens[i]] for i in range(nb.value)]

    def upload_by_ranges(self, boundaries):
        """uploads the (deferred) host inputs in key order, range after range; sub-jobs created afterwards start as soon as the blocks
        of their own range are on the device"""
        n = len(boundaries)
        keys = C.create_string_buffer(16 * max(1, n))
        lens = (C.c_uint32 * max(1, n))()
        for i, b in enumerate(boundaries):
            keys[16 * i:16 * i + len(b)] = b
            lens[i] = len(b)
        _check(lib().b200c_job_upload_by_ranges(self._h, keys, lens, n))

    def sub_job(self, range_start=None, range_end=None, **kw):
        """a job over this job's inputs (shared device copies) restricted to range_start <= user key < range_end"""
        merged = {k: v for k, v in self._kw.items() if k not in ("range_start", "range_end")}
        merged.update(kw)
        return CompactionJob(parent=self, range_start=range_start, range_end=range_end, **merged)

    def _wait_for_torch(self):
        """The library works on its own non-blocking streams: device tensors handed to it must be complete.  torch kernels that are
        still producing them (on torch's streams) are waited for here, as any caller of a stream-based C API has to."""
        if self._torch_device_inputs:
            import torch
            torch.cuda.synchronize(self.params.device)

    def add_input(self, data, level=0, file_number=0, deferred=False):
        """data: bytes (host image) or a CUDA uint8 torch tensor (device-resident image).  deferred: a host image whose upload waits
        for upload_by_ranges() (or the run)."""
        L = lib()
        host_kind = MEM_HOST_DEFERRED if deferred else MEM_HOST
        if isinstance(data, (bytes, bytearray)):
            buf = C.create_string_buffer(bytes(data), len(data))
            self._keep.append(buf)
            _check(L.b200c_job_add_input(self._h, level, file_number, C.cast(buf, C.c_void_p), len(data), host_kind))
        elif hasattr(data, "data_ptr"):
            self._keep.append(data)
            kind = MEM_DEVICE if data.is_cuda else host_kind
            self._torch_device_inputs = self._torch_device_inputs or bool(data.is_cuda)
            _check(L.b200c_job_add_input(self._h, level, file_number, C.c_void_p(data.data_ptr()), data.numel() * data.element_size(), kind))
        else:
            raise TypeError("input must be bytes or a torch tensor")
        self.ninputs += 1

    def run(self, until=3):
        L = lib()
        self._wait_for_torch()
        _check(L.b200c_job_run(self._h) if until == 3 else L.b200c_job_run_until(self._h, until))
        return self

    def encode_columns(self, n, pfx, tr, vref, meta):
        """TableBuilder side alone: device columns (torch CUDA tensors) -> BlockBasedTable image(s)."""
        self._keep += [pfx, tr, vref, meta]
        self._torch_device_inputs = True
        self._wait_for_torch()
        _check(lib().b200c_job_encode_columns(self._h, n, C.c_void_p(pfx.data_ptr()), C.c_void_p(tr.data_ptr()),
                                               C.c_void_p(vref.data_ptr()), C.c_void_p(meta.data_ptr())))
        return self

    def encode_kv(self, entries):
        """TableBuilder side with host records: entries = [(internal key bytes, value bytes)] in order -> BlockBasedTable image(s)"""
        import array
        arena = bytearray()
        offs, klens = array.array("Q"), array.array("I")
        for k, v in entries:
            offs.append(len(arena))
            klens.append(len(k))
            arena += k + v
        offs.append(len(arena))
        if not klens:
            klens.append(0)
        ab = (C.c_char * max(1, len(arena))).from_buffer(arena) if arena else (C.c_char * 1)()
        ob = (C.c_uint64 * len(offs)).from_buffer(offs)
        kb = (C.c_uint32 * len(klens)).from_buffer(klens)
        _check(lib().b200c_job_encode_kv(self._h, len(entries), ab, ob, kb))
        return self

    def kernel_times(self):
        """[(name, microseconds)] of the last run when created with profile=1"""
        L = lib()
        out = []
        for i in range(L.b200c_job_kernel_time_count(self._h)):
            name, us = C.c_char_p(), C.c_double()
            _check(L.b200c_job_kernel_time(self._h, i, C.byref(name), C.byref(us)))
            out.append((name.value.decode(), us.value))
        return out

    def stats(self):
        s = JobStats()
        _check(lib().b200c_job_get_stats(self._h, C.byref(s)))
        return s

    def output_count(self):
        n = lib().b200c_job_output_count(self._h)
        if n < 0:
            raise B200cError(-n, "job has not run")
        return n

    def output_meta(self, i):
        m = FileMeta()
        _check(lib().b200c_job_output_meta(self._h, i, C.byref(m)))
        return m

    def output_bytes(self, i):
        m = self.output_meta(i)
        buf = C.create_string_buffer(m.file_size)
        _check(lib().b200c_job_output_read(self._h, i, buf, m.file_size))
        return buf.raw

    def output_read_into(self, i, tensor):
        """copy output i into a preallocated uint8 torch tensor (host, or device when output_mem='device')"""
        m = self.output_meta(i)
        assert tensor.numel() >= m.file_size
        _check(lib().b200c_job_output_read(self._h, i, C.c_void_p(tensor.data_ptr()), tensor.numel()))
        return m.file_size

    def output_ptr(self, i):
        p, n = C.c_void_p(), C.c_uint64()
        _check(lib().b200c_job_output_data(self._h, i, C.byref(p), C.byref(n)))
        return p.value, n.value

    def outputs(self):
        return [self.output_bytes(i) for i in range(self.output_count())]

    def debug(self, what, run=0):
        L = lib()
        n = C.c_uint64()
        _check(L.b200c_job_debug_read(self._h, what, run, None, 0, C.byref(n)))
        buf = C.create_string_buffer(max(1, n.value))
        _check(L.b200c_job_debug_read(self._h, what, run, buf, n.value, C.byref(n)))
        return buf.raw[: n.value]

    def close(self):
        if self._h:
            lib().b200c_job_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
