"""zpaqfranz_b200 -- H100-native (sm_90a) implementation of zpaqfranz's block compressor and dedup
fragmenter hot paths, behind the reference's libzpaq API.

This package is a thin ctypes view of the C-ABI shared library (include/zq_b200.h).  The compute is
hand-written CUDA inside libzqb200.so; there is no CPU fallback: without the built library the import
fails, and without a CUDA device `Context()` raises.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.environ.get("ZQ_LIB", os.path.join(_HERE, "libzqb200.so"))   # ZQ_LIB: tuning builds (zpaqfranz_b200/build.py)

ZQ_OK, ZQ_E_NODEVICE, ZQ_E_ARG, ZQ_E_METHOD, ZQ_E_NOMEM, ZQ_E_OUTPUT, ZQ_E_UNSUPPORTED = 0, -1, -2, -3, -4, -5, -6


class ZqError(RuntimeError):
    """Raised where the reference would call libzpaq::error() (Z:12560)."""

    def __init__(self, code, msg):
        super().__init__("zq error %d: %s" % (code, msg))
        self.code = code


def _load():
    if not os.path.exists(_LIB_PATH):
        raise ImportError(
            "libzqb200.so is not built: run `python zpaqfranz_b200/build.py` "
            "(or __graft_entry__.build()). There is no CPU fallback.")
    lib = C.CDLL(_LIB_PATH)
    u8p, u32p, u64p, cpp = C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.POINTER(C.c_char_p)
    lib.zq_create.restype = C.c_void_p
    lib.zq_create.argtypes = [C.c_int]
    lib.zq_destroy.argtypes = [C.c_void_p]
    lib.zq_last_error.restype = C.c_char_p
    lib.zq_last_error.argtypes = [C.c_void_p]
    lib.zq_version.restype = C.c_char_p
    lib.zq_set_stream.argtypes = [C.c_void_p, C.c_void_p]
    lib.zq_compress_bound.restype = C.c_uint64
    lib.zq_compress_bound.argtypes = [C.c_uint32]
    lib.zq_plan_block.argtypes = [C.c_char_p, C.c_void_p, C.c_uint32, C.c_char_p, C.c_size_t, C.POINTER(C.c_int),
                                  C.c_void_p, u32p, C.c_void_p, u32p, C.c_char_p, C.c_size_t]
    for name in ("zq_compress_blocks", "zq_compress_blocks_device"):
        f = getattr(lib, name)
        f.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, cpp, cpp, cpp, C.c_int, C.c_int,
                      C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    lib.zq_decompress_blocks.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_uint64, C.c_void_p, C.c_void_p]
    lib.zq_decompress_blocks_ex.argtypes = lib.zq_decompress_blocks.argtypes + [C.c_void_p, C.c_void_p]
    lib.zq_decompress_prefix.argtypes = lib.zq_decompress_blocks.argtypes
    lib.zq_decompress_last_segments.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.zq_compress_segments.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_char_p, C.c_uint32,
                                         C.c_char_p, C.c_uint32, cpp, cpp, C.c_int, C.c_void_p, C.c_int,
                                         C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    lib.zq_fragment_ex.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_uint32,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
    lib.zq_add_files.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_char_p, C.c_int, C.c_char_p, C.c_uint32,
                                 C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p,
                                 C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    lib.zq_jit_context_source.argtypes = [C.c_void_p, C.c_uint32, C.c_char_p, C.c_uint32, u32p, C.c_char_p, C.c_size_t]
    lib.zq_jit_coder_source.argtypes = [C.c_void_p, C.c_uint32, C.c_char_p, C.c_uint32, u32p, C.c_char_p, C.c_size_t]
    lib.zq_jit_compile.argtypes = [C.c_char_p, u32p, C.c_char_p, C.c_size_t]
    lib.zq_file_sort_key.restype = C.c_uint64
    lib.zq_file_sort_key.argtypes = [C.c_char_p, C.c_int64]
    lib.zq_dedup_first.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    lib.zq_journal_header.argtypes = [C.c_void_p, C.c_char_p, C.c_int64, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p]
    lib.zq_journal_index.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    lib.zq_pipe_create.restype = C.c_void_p
    lib.zq_pipe_create.argtypes = [C.c_int, C.c_int]
    lib.zq_pipe_destroy.argtypes = [C.c_void_p]
    lib.zq_pipe_submit.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, cpp, cpp, cpp, C.c_int, C.c_int, C.c_int,
                                   C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    lib.zq_pipe_wait.argtypes = [C.c_void_p, C.c_int]
    lib.zq_pipe_last_error.restype = C.c_char_p
    lib.zq_pipe_last_error.argtypes = [C.c_void_p]
    lib.zq_pipe_launch_count.restype = C.c_uint64
    lib.zq_pipe_launch_count.argtypes = [C.c_void_p]
    lib.zq_model_config.restype = C.c_char_p
    lib.zq_model_config.argtypes = [C.c_int]
    lib.zq_assemble_config.argtypes = [C.c_char_p, C.POINTER(C.c_int), C.c_void_p, u32p, C.c_void_p, u32p, C.c_char_p, C.c_size_t,
                                       C.c_char_p, C.c_size_t]
    for name in ("zq_sha1", "zq_sha256", "zq_xxh3_128", "zq_blake3", "zq_sha1_device", "zq_crc32", "zq_xxh64", "zq_md5", "zq_sha3_256"):
        getattr(lib, name).argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.zq_fragment.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_uint32,
                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
    lib.zq_launch_count.restype = C.c_uint64
    lib.zq_launch_count.argtypes = [C.c_void_p]
    lib.zq_last_timings.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
    lib.zq_dist_create.restype = C.c_void_p
    lib.zq_dist_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.zq_dist_create_cb.restype = C.c_void_p
    lib.zq_dist_create_cb.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    lib.zq_dist_destroy.argtypes = [C.c_void_p]
    lib.zq_dist_last_error.restype = C.c_char_p
    lib.zq_dist_last_error.argtypes = [C.c_void_p]
    lib.zq_dist_bytes_exchanged.restype = C.c_uint64
    lib.zq_dist_bytes_exchanged.argtypes = [C.c_void_p]
    lib.zq_dist_unique_id.argtypes = [C.c_void_p]
    lib.zq_dist_shard_range.argtypes = [C.c_uint64, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    lib.zq_dist_shard_lpt.argtypes = [C.c_void_p, C.c_uint64, C.c_int, C.c_void_p]
    lib.zq_dist_exchange_sizes.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    lib.zq_dist_dedup.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    lib.zq_dist_stitch_fragments.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p]
    lib.zq_last_timings_ex.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.c_int]
    lib.zq_suffix_array.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
    return lib


lib = _load()

TIMING_KEYS = ("total", "sha1", "sufsort", "lzparse", "frame", "model", "h2d", "d2h")
TIMING_KEYS_EX = TIMING_KEYS + ("lz_scan0", "lz_scan1", "lz_walk", "lz_emit")


def plan_block(method, data=b""):
    """Host-side planning (== the part of libzpaq::compressBlock before the data is touched).
    Returns dict(method=expanded, args=[9], header=bytes, pcomp=bytes)."""
    data = bytes(data)
    exp = C.create_string_buffer(1024)
    args = (C.c_int * 9)()
    hdr = C.create_string_buffer(70000)
    pc = C.create_string_buffer(70000)
    hl, pl = C.c_uint32(70000), C.c_uint32(70000)
    err = C.create_string_buffer(512)
    rc = lib.zq_plan_block(method.encode(), data, len(data), exp, 1024, args, hdr, C.byref(hl), pc, C.byref(pl), err, 512)
    if rc:
        raise ZqError(rc, err.value.decode(errors="replace"))
    return dict(method=exp.value.decode(), args=list(args), header=hdr.raw[:hl.value], pcomp=pc.raw[:pl.value])


def file_sort_key(path, size):
    """The key Jidac::add sorts the files to add by (then by path): extension bytes, then descending size."""
    return int(lib.zq_file_sort_key(path.encode() if isinstance(path, str) else path, int(size)))


def model_config(level):
    """ZPAQL source of the built-in model Compressor::startBlock(level) selects (1 min.cfg, 2 mid.cfg) or None."""
    r = lib.zq_model_config(int(level))
    return r.decode() if r else None


def assemble_config(config, args=None):
    """== libzpaq::Compiler: ZPAQL source -> dict(header=bytes, pcomp=bytes, pcomp_cmd=str). No GPU needed."""
    a = (C.c_int * 9)(*(list(args or []) + [0] * 9)[:9])
    hdr = C.create_string_buffer(70000)
    pc = C.create_string_buffer(70000)
    cmd = C.create_string_buffer(4096)
    hl, pl = C.c_uint32(70000), C.c_uint32(70000)
    err = C.create_string_buffer(512)
    rc = lib.zq_assemble_config(config.encode() if isinstance(config, str) else config, a, hdr, C.byref(hl), pc, C.byref(pl),
                                cmd, 4096, err, 512)
    if rc:
        raise ZqError(rc, err.value.decode(errors="replace"))
    return dict(header=hdr.raw[:hl.value], pcomp=pc.raw[:pl.value], pcomp_cmd=cmd.value.decode())


def _cstr_array(v, n, uniform):
    if v is None:
        return None
    if isinstance(v, (str, bytes)):
        v = [v]
    arr = (C.c_char_p * len(v))(*[(s.encode() if isinstance(s, str) else s) for s in v])
    return arr


ALLGATHER_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t)


def shard_range(total, rank, world):
    lo, hi = C.c_uint64(0), C.c_uint64(0)
    lib.zq_dist_shard_range(int(total), int(rank), int(world), C.byref(lo), C.byref(hi))
    return int(lo.value), int(hi.value)


def shard_lpt(costs, world):
    """owner[i] of every unit, longest first onto the least loaded rank (zq_dist_shard_lpt)."""
    c = np.ascontiguousarray(costs, dtype=np.uint64)
    owner = np.zeros(len(c), dtype=np.int32)
    if len(c):
        lib.zq_dist_shard_lpt(c.ctypes.data, len(c), int(world), owner.ctypes.data)
    return owner


def dist_unique_id():
    """Rank 0: the 128 bytes every rank passes to Dist(...) (ncclGetUniqueId)."""
    buf = (C.c_uint8 * 128)()
    rc = lib.zq_dist_unique_id(buf)
    if rc:
        raise ZqError(rc, lib.zq_dist_last_error(None).decode(errors="replace"))
    return bytes(buf)


class ZqStitch(C.Structure):
    _fields_ = [("first_keep", C.c_uint64), ("n_keep", C.c_uint64), ("global_first", C.c_uint64), ("global_total", C.c_uint64),
                ("begin", C.c_uint64), ("end", C.c_uint64), ("restart_at", C.c_uint64), ("again", C.c_int32), ("restart", C.c_int32)]


class Dist:
    """The exchanges of a multi-GPU run (zq_dist_*): NCCL when unique_id is given, a Python all-gather callable
    `allgather(in_bytes) -> list of world bytes objects` otherwise (CPU tests over gloo), nothing for world == 1."""

    def __init__(self, device, rank, world, unique_id=None, allgather=None):
        self.rank, self.world = int(rank), int(world)
        self._cb = None
        if allgather is not None and world > 1:
            def cb(user, pin, pout, nbytes):
                try:
                    parts = allgather(C.string_at(pin, nbytes))
                    C.memmove(pout, b"".join(parts), nbytes * self.world)
                    return 0
                except Exception:
                    return 1
            self._cb = ALLGATHER_FN(cb)
            self._h = lib.zq_dist_create_cb(self.rank, self.world, C.cast(self._cb, C.c_void_p), None)
        else:
            idb = (C.c_uint8 * 128)(*unique_id) if (unique_id is not None and world > 1) else None
            self._h = lib.zq_dist_create(int(device), self.rank, self.world, idb)
        if not self._h:
            raise ZqError(ZQ_E_NODEVICE, lib.zq_dist_last_error(None).decode(errors="replace"))

    def close(self):
        if self._h:
            lib.zq_dist_destroy(self._h)
            self._h = None

    def _check(self, rc):
        if rc:
            raise ZqError(rc, lib.zq_dist_last_error(self._h).decode(errors="replace"))

    def exchange_sizes(self, local_sizes, total):
        """(all_sizes u32[total], offsets u64[total]) from every rank's contiguous shard of compressed sizes."""
        loc = np.ascontiguousarray(local_sizes, dtype=np.uint32)
        sizes = np.zeros(int(total), dtype=np.uint32)
        offs = np.zeros(int(total), dtype=np.uint64)
        self._check(lib.zq_dist_exchange_sizes(self._h, loc.ctypes.data if len(loc) else None, int(total),
                                               sizes.ctypes.data if total else None, offs.ctypes.data if total else None))
        return sizes, offs

    def dedup(self, digests):
        """digests u8[n,20] of this rank's fragments in archive order -> (is_first bool[n], unique fragments of all ranks)."""
        dg = np.ascontiguousarray(digests, dtype=np.uint8).reshape(-1, 20)
        first = np.zeros(len(dg), dtype=np.uint8)
        uniq = C.c_uint64(0)
        self._check(lib.zq_dist_dedup(self._h, dg.ctypes.data if len(dg) else None, len(dg), first.ctypes.data if len(dg) else None, C.byref(uniq)))
        return first.astype(bool), int(uniq.value)

    def stitch_fragments(self, stream_total, lo, hi, start, avail_end, frag_len):
        """One stream cut across the ranks (zq_dist_stitch_fragments): this rank fragmented [start, avail_end) into
        frag_len.  Returns the zq_stitch record as a dict."""
        fl = np.ascontiguousarray(frag_len, dtype=np.uint32)
        st = ZqStitch()
        self._check(lib.zq_dist_stitch_fragments(self._h, int(stream_total), int(lo), int(hi), int(start), int(avail_end),
                                                 fl.ctypes.data if len(fl) else None, len(fl), C.byref(st)))
        return {k: int(getattr(st, k)) for k, _ in ZqStitch._fields_}

    def bytes_exchanged(self):
        return int(lib.zq_dist_bytes_exchanged(self._h))


class Pipe:
    """`depth` batches in flight on one device (zq_pipe_*): submit() returns a ticket, wait(ticket) the
    (out_off, out_len) of that batch.  Buffers passed to submit() must stay alive until wait()."""

    def __init__(self, device=0, depth=2):
        self._h = lib.zq_pipe_create(int(device), int(depth))
        if not self._h:
            raise ZqError(ZQ_E_NODEVICE, lib.zq_last_error(None).decode(errors="replace"))
        self._keep = {}

    def close(self):
        if self._h:
            lib.zq_pipe_destroy(self._h)
            self._h = None

    def submit(self, in_ptr, offsets, lengths, out_ptr, out_cap, method="2", filename=None, comment=None, dosha1=True, device=False):
        """in_ptr/out_ptr: integer addresses (host, or device when device=True)."""
        off = np.ascontiguousarray(offsets, dtype=np.uint64)
        ln = np.ascontiguousarray(lengths, dtype=np.uint32)
        n = len(off)
        m, f, cm = _cstr_array(method, n, True), _cstr_array(filename, n, True), _cstr_array(comment, n, True)
        ooff = np.zeros(n, dtype=np.uint64)
        olen = np.zeros(n, dtype=np.uint32)
        t = lib.zq_pipe_submit(self._h, n, in_ptr, off.ctypes.data, ln.ctypes.data, m, f, cm, 1, 1 if dosha1 else 0,
                               1 if device else 0, out_ptr, out_cap, ooff.ctypes.data, olen.ctypes.data)
        if t < 0:
            raise ZqError(t, "submit failed")
        self._keep[t] = (off, ln, m, f, cm, ooff, olen)
        return t

    def wait(self, ticket):
        rc = lib.zq_pipe_wait(self._h, int(ticket))
        keep = self._keep.pop(ticket)
        if rc:
            raise ZqError(rc, lib.zq_pipe_last_error(self._h).decode(errors="replace"))
        return keep[5], keep[6]

    def launch_count(self):
        return int(lib.zq_pipe_launch_count(self._h))


class Context:
    """One CUDA device context (== one libzpaq Compressor-owning thread)."""

    def __init__(self, device=0):
        self._h = lib.zq_create(int(device))
        if not self._h:
            raise ZqError(ZQ_E_NODEVICE, lib.zq_last_error(None).decode(errors="replace"))

    def close(self):
        if self._h:
            lib.zq_destroy(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc:
            raise ZqError(rc, lib.zq_last_error(self._h).decode(errors="replace"))

    def set_stream(self, cuda_stream_ptr):
        """Issue this context's work on the given cudaStream_t (int), e.g. torch.cuda.current_stream().cuda_stream."""
        self._check(lib.zq_set_stream(self._h, cuda_stream_ptr))

    # -- block compression ------------------------------------------------------------------------
    def compress_blocks(self, arena, offsets, lengths, method="2", filename=None, comment=None, dosha1=True, out=None):
        """Element-wise libzpaq::compressBlock over units arena[offsets[i]:offsets[i]+lengths[i]].
        `arena` is a contiguous uint8 numpy array (pinned or pageable host memory).
        method/filename/comment: one string for all units, or a list per unit.
        Returns (out_array, out_off, out_len)."""
        arena = np.ascontiguousarray(arena, dtype=np.uint8)
        off = np.ascontiguousarray(offsets, dtype=np.uint64)
        ln = np.ascontiguousarray(lengths, dtype=np.uint32)
        n = len(off)
        uniform = all(isinstance(x, (str, bytes)) or x is None for x in (method, filename, comment))
        if not uniform:
            def expand(x):
                return [x] * n if isinstance(x, (str, bytes)) else x
            method, filename, comment = expand(method), expand(filename), expand(comment)
        m, f, cm = _cstr_array(method, n, uniform), _cstr_array(filename, n, uniform), _cstr_array(comment, n, uniform)
        if out is None:
            cap = int(sum(int(lib.zq_compress_bound(int(x))) for x in np.unique(ln)) if n < 64 else
                      int(lib.zq_compress_bound(int(ln.max()))) * n)
            out = np.empty(cap, dtype=np.uint8)
        ooff = np.zeros(n, dtype=np.uint64)
        olen = np.zeros(n, dtype=np.uint32)
        rc = lib.zq_compress_blocks(self._h, n, arena.ctypes.data, off.ctypes.data, ln.ctypes.data, m, f, cm,
                                    1 if uniform else 0, 1 if dosha1 else 0, out.ctypes.data, out.size,
                                    ooff.ctypes.data, olen.ctypes.data)
        self._check(rc)
        return out, ooff, olen

    def compress_blocks_device(self, d_in_ptr, offsets, lengths, d_out_ptr, out_cap, method="2", filename=None,
                               comment=None, dosha1=True):
        """Same, with device pointers (ints) for the input arena and the output buffer."""
        off = np.ascontiguousarray(offsets, dtype=np.uint64)
        ln = np.ascontiguousarray(lengths, dtype=np.uint32)
        n = len(off)
        m, f, cm = _cstr_array(method, n, True), _cstr_array(filename, n, True), _cstr_array(comment, n, True)
        ooff = np.zeros(n, dtype=np.uint64)
        olen = np.zeros(n, dtype=np.uint32)
        rc = lib.zq_compress_blocks_device(self._h, n, d_in_ptr, off.ctypes.data, ln.ctypes.data, m, f, cm, 1,
                                           1 if dosha1 else 0, d_out_ptr, out_cap, ooff.ctypes.data, olen.ctypes.data)
        self._check(rc)
        return ooff, olen

    def compress_block(self, data, method="1", filename=None, comment=None, dosha1=True):
        """Single-block convenience: bytes in, one ZPAQ block out (== compressBlock)."""
        a = np.frombuffer(bytes(data), dtype=np.uint8) if len(data) else np.zeros(0, dtype=np.uint8)
        out, ooff, olen = self.compress_blocks(a if len(a) else np.zeros(1, np.uint8), [0], [len(data)], method, filename, comment, dosha1)
        return out[: int(olen[0])].tobytes()

    def compress_segments(self, arena, offsets, lengths, header, pcomp=b"", filename=None, comment=None, sha1=None, tag=True):
        """libzpaq::Compressor driven directly, once per unit, with the caller's model: `header` is the stored block
        header, `pcomp` the PCOMP bytecode to announce, `sha1` an (n,20) array of digests to store or None.
        Returns (out_array, out_off, out_len)."""
        arena = np.ascontiguousarray(arena, dtype=np.uint8)
        off = np.ascontiguousarray(offsets, dtype=np.uint64)
        ln = np.ascontiguousarray(lengths, dtype=np.uint32)
        n = len(off)
        fn = _cstr_array(filename, n, True)
        cm = _cstr_array(comment, n, True)
        uniform = 1 if all(x is None or len(x) == 1 for x in (fn, cm)) else 0
        dg = None if sha1 is None else np.ascontiguousarray(sha1, dtype=np.uint8).reshape(n, 20)
        cap = int(sum(int(lib.zq_compress_bound(int(x))) for x in ln)) + n * (2 * len(pcomp) + len(header))
        out = np.empty(cap, dtype=np.uint8)
        ooff = np.zeros(n, dtype=np.uint64)
        olen = np.zeros(n, dtype=np.uint32)
        self._check(lib.zq_compress_segments(self._h, n, arena.ctypes.data, off.ctypes.data, ln.ctypes.data, bytes(header), len(header),
                                             bytes(pcomp) if pcomp else None, len(pcomp), fn, cm, uniform,
                                             dg.ctypes.data if dg is not None else None, 1 if tag else 0,
                                             out.ctypes.data, out.size, ooff.ctypes.data, olen.ctypes.data))
        return out, ooff, olen

    def decompress_blocks(self, arena, offsets, lengths, expect_len=None, out_cap=None, details=False):
        """Element-wise libzpaq::decompress of complete blocks arena[offsets[i]:+lengths[i]].
        Returns (out_array, out_off, out_len); with details=True also (in_used, trailers[n,21])."""
        arena = np.ascontiguousarray(arena, dtype=np.uint8)
        off = np.ascontiguousarray(offsets, dtype=np.uint64)
        ln = np.ascontiguousarray(lengths, dtype=np.uint32)
        n = len(off)
        ex = None if expect_len is None else np.ascontiguousarray(expect_len, dtype=np.uint32)
        if out_cap is None:
            out_cap = int(ex.sum()) if ex is not None else int(ln.sum()) * 64 + (1 << 20)
        out = np.empty(max(out_cap, 1), dtype=np.uint8)
        ooff = np.zeros(n, dtype=np.uint64)
        olen = np.zeros(n, dtype=np.uint32)
        if details:
            used = np.zeros(n, dtype=np.uint32)
            tr = np.zeros((n, 21), dtype=np.uint8)
            self._check(lib.zq_decompress_blocks_ex(self._h, n, arena.ctypes.data, off.ctypes.data, ln.ctypes.data,
                                                    ex.ctypes.data if ex is not None else None, out.ctypes.data, out.size,
                                                    ooff.ctypes.data, olen.ctypes.data, used.ctypes.data, tr.ctypes.data))
            return out, ooff, olen, used, tr
        self._check(lib.zq_decompress_blocks(self._h, n, arena.ctypes.data, off.ctypes.data, ln.ctypes.data,
                                             ex.ctypes.data if ex is not None else None, out.ctypes.data, out.size,
                                             ooff.ctypes.data, olen.ctypes.data))
        return out, ooff, olen

    def decompress_prefix(self, arena, offsets, lengths, max_out):
        """The first max_out[i] bytes of every block (zq_decompress_prefix).  Returns (out, out_off, out_len)."""
        arena = np.ascontiguousarray(arena, dtype=np.uint8)
        off = np.ascontiguousarray(offsets, dtype=np.uint64)
        ln = np.ascontiguousarray(lengths, dtype=np.uint32)
        mx = np.ascontiguousarray(max_out, dtype=np.uint32)
        n = len(off)
        out = np.empty(max(int(mx.sum()), 1), dtype=np.uint8)
        ooff = np.zeros(n, dtype=np.uint64)
        olen = np.zeros(n, dtype=np.uint32)
        self._check(lib.zq_decompress_prefix(self._h, n, arena.ctypes.data, off.ctypes.data, ln.ctypes.data, mx.ctypes.data,
                                             out.ctypes.data, out.size, ooff.ctypes.data, olen.ctypes.data))
        return out, ooff, olen

    # -- hashes -------------------------------------------------------------------------------------
    def _hash(self, fn, dlen, arena, offsets, lengths):
        arena = np.ascontiguousarray(arena, dtype=np.uint8)
        off = np.ascontiguousarray(offsets, dtype=np.uint64)
        ln = np.ascontiguousarray(lengths, dtype=np.uint64)
        out = np.zeros((len(off), dlen), dtype=np.uint8)
        self._check(fn(self._h, len(off), arena.ctypes.data, off.ctypes.data, ln.ctypes.data, out.ctypes.data))
        return out

    def sha1(self, arena, offsets, lengths):
        return self._hash(lib.zq_sha1, 20, arena, offsets, lengths)

    def sha256(self, arena, offsets, lengths):
        return self._hash(lib.zq_sha256, 32, arena, offsets, lengths)

    def xxh3_128(self, arena, offsets, lengths):
        return self._hash(lib.zq_xxh3_128, 16, arena, offsets, lengths)

    def blake3(self, arena, offsets, lengths):
        return self._hash(lib.zq_blake3, 32, arena, offsets, lengths)

    def md5(self, arena, offsets, lengths):
        return self._hash(lib.zq_md5, 16, arena, offsets, lengths)

    def sha3_256(self, arena, offsets, lengths):
        return self._hash(lib.zq_sha3_256, 32, arena, offsets, lengths)

    def crc32(self, arena, offsets, lengths):
        """CRC-32 per buffer as little-endian bytes (4 per row)."""
        return self._hash(lib.zq_crc32, 4, arena, offsets, lengths)

    def xxh64(self, arena, offsets, lengths):
        """XXH64 (seed 0) per buffer as little-endian bytes (8 per row)."""
        return self._hash(lib.zq_xxh64, 8, arena, offsets, lengths)

    def add_files(self, arena, offsets, lengths, method="1", fragment=6, date14="20260101000000", first_id=1):
        """The archiver's add loop over files in memory (== Jidac::add's data path for a fresh archive): returns
        dict(d=bytes of the data blocks, h=bytes of the fragment-table blocks, file_frags=[ids per file], nblocks)."""
        arena = np.ascontiguousarray(arena, dtype=np.uint8)
        off = np.ascontiguousarray(offsets, dtype=np.uint64)
        ln = np.ascontiguousarray(lengths, dtype=np.uint64)
        n = len(off)
        total = int(ln.sum())
        dcap = total + total // 8 + (1 << 20) + 70000 * (total // 4096 + n + 4)
        dcap = min(dcap, total * 2 + (64 << 20))
        d = np.empty(dcap, dtype=np.uint8)
        hcap = (total // 4096 + n + 16) * 64 + (1 << 20)
        h = np.empty(hcap, dtype=np.uint8)
        dl, hl = C.c_uint64(0), C.c_uint64(0)
        idcap = total // 4096 + n + 16
        ids = np.zeros(idcap, dtype=np.uint32)
        first = np.zeros(n + 1, dtype=np.uint64)
        nb = C.c_uint32(0)
        self._check(lib.zq_add_files(self._h, n, arena.ctypes.data, off.ctypes.data, ln.ctypes.data, method.encode(), int(fragment),
                                     date14.encode(), int(first_id), d.ctypes.data, d.size, C.byref(dl), h.ctypes.data, h.size,
                                     C.byref(hl), ids.ctypes.data, ids.size, first.ctypes.data, C.byref(nb)))
        return dict(d=d[: dl.value].tobytes(), h=h[: hl.value].tobytes(), nblocks=nb.value,
                    file_frags=[ids[int(first[i]): int(first[i + 1])].tolist() for i in range(n)])

    def last_segments(self):
        """(block, out_begin, out_end, trailer offset) of every segment of the last decompress call."""
        p, n = C.c_void_p(0), C.c_uint64(0)
        self._check(lib.zq_decompress_last_segments(self._h, C.byref(p), C.byref(n)))
        if not n.value:
            return []
        a = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint32)), shape=(n.value, 4))
        return [tuple(int(x) for x in row) for row in a]

    def dedup_first(self, sha1):
        """first[i] = earliest fragment with the digest of fragment i (the device fragment index); sha1: (n, 20) uint8."""
        dg = np.ascontiguousarray(sha1, dtype=np.uint8).reshape(-1, 20)
        first = np.zeros(len(dg), dtype=np.uint32)
        self._check(lib.zq_dedup_first(self._h, len(dg), dg.ctypes.data, first.ctypes.data))
        return first

    def journal_header(self, date14, cdata, htsize):
        """The transaction's "c" block (writeJidacHeader): bytes."""
        out = np.empty(4096, dtype=np.uint8)
        n = C.c_uint64(0)
        self._check(lib.zq_journal_header(self._h, date14.encode(), int(cdata), int(htsize), out.ctypes.data, out.size, C.byref(n)))
        return out[: n.value].tobytes()

    def journal_index(self, date14, records):
        """The transaction's "i" blocks from records (date, name: bytes, attr: bytes, fragment ids): (bytes, nblocks)."""
        nrec = len(records)
        dates = np.array([r[0] for r in records], dtype=np.int64)
        names = (C.c_char_p * max(nrec, 1))(*[bytes(r[1]) for r in records])
        attrs = [bytes(r[2]) if r[0] else b"" for r in records]
        ab = np.frombuffer(b"".join(attrs) + b"\0", dtype=np.uint8)
        al = np.array([len(a) for a in attrs], dtype=np.uint32)
        ao = (np.cumsum(al, dtype=np.uint64) - al).astype(np.uint64)
        fr = [list(r[3]) if r[0] else [] for r in records]
        ff = np.concatenate([[0], np.cumsum([len(f) for f in fr])]).astype(np.uint64)
        fa = np.array([x for f in fr for x in f] + [0], dtype=np.uint32)
        total = sum(len(r[1]) + 17 for r in records) + int(al.sum()) + 4 * fa.size
        out = np.empty(total * 2 + 4096 * (total // 16000 + 2), dtype=np.uint8)
        n, nb = C.c_uint64(0), C.c_uint32(0)
        self._check(lib.zq_journal_index(self._h, date14.encode(), nrec, dates.ctypes.data, names, ab.ctypes.data, ao.ctypes.data,
                                         al.ctypes.data, ff.ctypes.data, fa.ctypes.data, out.ctypes.data, out.size, C.byref(n), C.byref(nb)))
        return out[: n.value].tobytes(), nb.value

    # -- fragmenter ---------------------------------------------------------------------------------
    def fragment(self, arena, offsets, lengths, fragment=6, blocksize=(1 << 26) - 4096, want_sha1=True):
        arena = np.ascontiguousarray(arena, dtype=np.uint8)
        off = np.ascontiguousarray(offsets, dtype=np.uint64)
        ln = np.ascontiguousarray(lengths, dtype=np.uint64)
        nf = len(off)
        minf = min(64 << fragment, blocksize - 12)
        cap = int(sum(int(x) // minf + 2 for x in ln))
        fl = np.zeros(cap, dtype=np.uint32)
        fh = np.zeros(cap, dtype=np.uint32)
        fs = np.zeros((cap, 20), dtype=np.uint8) if want_sha1 else None
        first = np.zeros(nf + 1, dtype=np.uint64)
        self._check(lib.zq_fragment(self._h, nf, arena.ctypes.data, off.ctypes.data, ln.ctypes.data, fragment, blocksize,
                                    fl.ctypes.data, fh.ctypes.data, fs.ctypes.data if want_sha1 else None, cap,
                                    first.ctypes.data))
        k = int(first[nf])
        return fl[:k], fh[:k], (fs[:k] if want_sha1 else None), first

    # -- introspection ------------------------------------------------------------------------------
    def launch_count(self):
        return int(lib.zq_launch_count(self._h))

    def last_timings(self, ex=False):
        if ex:
            ms = (C.c_float * 12)()
            lib.zq_last_timings_ex(self._h, ms, 12)
            return dict(zip(TIMING_KEYS_EX, [float(x) for x in ms]))
        ms = (C.c_float * 8)()
        lib.zq_last_timings(self._h, ms)
        return dict(zip(TIMING_KEYS, [float(x) for x in ms]))

    def suffix_array(self, data):
        a = np.frombuffer(bytes(data), dtype=np.uint8)
        sa = np.zeros(len(a), dtype=np.uint32)
        if len(a):
            self._check(lib.zq_suffix_array(self._h, a.ctypes.data, len(a), sa.ctypes.data))
        return sa
