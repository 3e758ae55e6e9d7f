"""ctypes views of the two CHECKERS under oracle/_ref/ (test infrastructure; never used by the product)."""
import ctypes as C
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")


class Oracle:
    def __init__(self, lib):
        self.lib = lib
        lib.zqo_lz_stream.restype = C.c_longlong
        lib.zqo_block_unmodeled.restype = C.c_longlong
        lib.zqo_fragment.restype = C.c_longlong
        lib.zqo_block_modeled.restype = C.c_longlong

    def sha1(self, data):
        out = C.create_string_buffer(20)
        self.lib.zqo_sha1(bytes(data), C.c_uint64(len(data)), out)
        return out.raw

    def suffix_array(self, data):
        data = bytes(data)
        sa = np.zeros(max(len(data), 1), dtype=np.uint32)
        self.lib.zqo_suffix_array(data, sa.ctypes.data_as(C.c_void_p), C.c_uint32(len(data)))
        return sa[: len(data)]

    def lz_stream(self, data, args, sa=None, tokens=False):
        data = bytes(data)
        a = (C.c_int * 9)(*args)
        cap = len(data) + len(data) // 16 + 1024
        out = C.create_string_buffer(cap)
        tok = np.zeros(3 * (len(data) + 1), dtype=np.uint32)
        ntok = C.c_uint64(0)
        sap = sa.ctypes.data_as(C.c_void_p) if sa is not None else None
        r = self.lib.zqo_lz_stream(data, C.c_uint32(len(data)), a, sap, out, C.c_uint64(cap),
                                   tok.ctypes.data_as(C.c_void_p), C.c_uint64(tok.size), C.byref(ntok))
        if r < 0:
            raise RuntimeError("zqo_lz_stream failed %d" % r)
        if tokens:
            return out.raw[:r], tok[: 3 * ntok.value].reshape(-1, 3)
        return out.raw[:r]

    def e8e9(self, data):
        b = C.create_string_buffer(bytes(data), len(data))
        self.lib.zqo_e8e9(b, C.c_int(len(data)))
        return b.raw

    def block_unmodeled(self, header, pcomp, filename, comment_full, stream, sha1):
        cap = len(stream) + len(stream) // 1000 + len(header) + len(pcomp) + 1024
        out = C.create_string_buffer(cap)
        r = self.lib.zqo_block_unmodeled(bytes(header), C.c_uint32(len(header)), bytes(pcomp), C.c_uint32(len(pcomp)),
                                         filename, comment_full, bytes(stream), C.c_uint64(len(stream)), sha1, out,
                                         C.c_uint64(cap))
        if r < 0:
            raise RuntimeError("zqo_block_unmodeled failed %d" % r)
        return out.raw[:r]

    def block_modeled(self, header, pcomp, filename, comment_full, stream, sha1):
        cap = len(stream) + len(stream) // 8 + len(header) + len(pcomp) + 4096
        out = C.create_string_buffer(cap)
        r = self.lib.zqo_block_modeled(bytes(header), C.c_uint32(len(header)), bytes(pcomp), C.c_uint32(len(pcomp)),
                                       filename, comment_full, bytes(stream), C.c_uint64(len(stream)), sha1, out,
                                       C.c_uint64(cap))
        if r < 0:
            raise RuntimeError("zqo_block_modeled failed %d" % r)
        return out.raw[:r]

    def table_sums(self):
        a, b = C.c_uint32(0), C.c_uint32(0)
        self.lib.zqo_table_sums(C.byref(a), C.byref(b))
        return a.value, b.value

    def fragment(self, data, fragment=6, blocksize=(1 << 26) - 4096):
        data = bytes(data)
        cap = len(data) // 64 + 16
        fl = np.zeros(cap, dtype=np.uint32)
        fh = np.zeros(cap, dtype=np.uint32)
        k = self.lib.zqo_fragment(data, C.c_uint64(len(data)), C.c_int(fragment), C.c_uint32(blocksize),
                                  fl.ctypes.data_as(C.c_void_p), fh.ctypes.data_as(C.c_void_p), C.c_uint64(cap))
        return fl[:k].copy(), fh[:k].copy()


class Ref:
    """The unmodified reference (libzpaq inside zpaqfranz.cpp) behind oracle/ref_shim.cpp."""

    def __init__(self, lib):
        self.lib = lib
        for f in ("zref_compress_block", "zref_decompress", "zref_lz_stream", "zref_fragment", "zref_compress_units_mt", "zref_compress_segment"):
            getattr(lib, f).restype = C.c_longlong
        lib.zref_last_error.restype = C.c_char_p

    def compress_block(self, data, method, filename=None, comment=None, dosha1=True):
        data = bytes(data)
        cap = len(data) + len(data) // 8 + 100000
        out = C.create_string_buffer(cap)
        fn = filename.encode() if isinstance(filename, str) else filename
        cm = comment.encode() if isinstance(comment, str) else comment
        r = self.lib.zref_compress_block(data, C.c_uint(len(data)), method.encode(), fn, cm, C.c_int(1 if dosha1 else 0),
                                         out, C.c_ulonglong(cap))
        if r < 0:
            raise RuntimeError("reference compressBlock failed: %s" % self.lib.zref_last_error().decode(errors="replace"))
        return out.raw[:r]

    def compress_segment(self, data, header=None, level=0, pcomp=b"", filename=None, comment=None, sha1=None, tag=True):
        """libzpaq::Compressor driven directly: writeTag/startBlock(level | header)/startSegment/postProcess/compress/
        endSegment(sha1)/endBlock."""
        data = bytes(data)
        cap = len(data) + len(data) // 8 + 200000
        out = C.create_string_buffer(cap)
        fn = filename.encode() if isinstance(filename, str) else filename
        cm = comment.encode() if isinstance(comment, str) else comment
        r = self.lib.zref_compress_segment(C.c_int(level), bytes(header) if header else None, bytes(pcomp) if pcomp else None,
                                           C.c_int(len(pcomp)), data, C.c_uint(len(data)), fn, cm,
                                           bytes(sha1) if sha1 is not None else None, C.c_int(1 if tag else 0), out, C.c_ulonglong(cap))
        if r < 0:
            raise RuntimeError("reference Compressor failed: %s" % self.lib.zref_last_error().decode(errors="replace"))
        return out.raw[:r]

    def compress_multi(self, segments, header=None, level=0, pcomp=b"", filename="seg", comment="", sha=True):
        """One block with several segments through the reference's Compressor class."""
        import numpy as _np
        data = b"".join(bytes(x) for x in segments)
        lens = _np.array([len(x) for x in segments], dtype=_np.uint32)
        offs = (_np.cumsum(lens, dtype=_np.uint64) - lens).astype(_np.uint64)
        cap = len(data) + len(data) // 8 + 200000 + 400 * len(segments)
        out = C.create_string_buffer(cap)
        self.lib.zref_compress_multi.restype = C.c_longlong
        r = self.lib.zref_compress_multi(C.c_int(level), bytes(header) if header else None, bytes(pcomp) if pcomp else None,
                                         C.c_int(len(pcomp)), C.c_int(len(segments)), data + b"\0", offs.ctypes.data_as(C.c_void_p),
                                         lens.ctypes.data_as(C.c_void_p), filename.encode(), comment.encode(), C.c_int(1 if sha else 0),
                                         out, C.c_ulonglong(cap))
        if r < 0:
            raise RuntimeError("reference Compressor failed: %s" % self.lib.zref_last_error().decode(errors="replace"))
        return out.raw[:r]

    def decompress(self, blob, cap):
        out = C.create_string_buffer(cap + 16)
        r = self.lib.zref_decompress(bytes(blob), C.c_ulonglong(len(blob)), out, C.c_ulonglong(cap + 16))
        if r < 0:
            raise RuntimeError("reference decompress failed: %s" % self.lib.zref_last_error().decode(errors="replace"))
        return out.raw[:r]

    def _digest(self, fn, n, data):
        out = C.create_string_buffer(n)
        fn(bytes(data), C.c_ulonglong(len(data)), out)
        return out.raw

    def sha1(self, d):
        return self._digest(self.lib.zref_sha1, 20, d)

    def sha256(self, d):
        return self._digest(self.lib.zref_sha256, 32, d)

    def xxh3_128(self, d):
        return self._digest(self.lib.zref_xxh3_128, 16, d)

    def blake3(self, d):
        return self._digest(self.lib.zref_blake3, 32, d)

    def md5(self, d):
        return self._digest(self.lib.zref_md5, 16, d)

    def sha3_256(self, d):
        return self._digest(self.lib.zref_sha3_256, 32, d)

    def xxh64(self, d):
        return self._digest(self.lib.zref_xxh64, 8, d)

    def crc32(self, d):
        return self._digest(self.lib.zref_crc32, 4, d)

    def divsufsort(self, data):
        data = bytes(data)
        sa = np.zeros(max(len(data), 1), dtype=np.int32)
        self.lib.zref_divsufsort(data, sa.ctypes.data_as(C.c_void_p), C.c_int(len(data)))
        return sa[: len(data)].astype(np.uint32)

    def make_config(self, method):
        args = (C.c_int * 9)()
        out = C.create_string_buffer(1 << 16)
        r = self.lib.zref_make_config(method.encode(), args, out, 1 << 16)
        if r < 0:
            raise RuntimeError(self.lib.zref_last_error().decode(errors="replace"))
        return out.value.decode(), list(args)

    def compile(self, config, args):
        a = (C.c_int * 9)(*args)
        hdr = C.create_string_buffer(70000)
        pc = C.create_string_buffer(70000)
        hl, pl = C.c_int(0), C.c_int(0)
        r = self.lib.zref_compile(config.encode(), a, hdr, C.byref(hl), pc, C.byref(pl))
        if r < 0:
            raise RuntimeError(self.lib.zref_last_error().decode(errors="replace"))
        return hdr.raw[: hl.value], pc.raw[: pl.value]

    def lz_stream(self, data, args):
        data = bytes(data)
        a = (C.c_int * 9)(*args)
        cap = len(data) + len(data) // 16 + 1024
        out = C.create_string_buffer(cap)
        r = self.lib.zref_lz_stream(data, C.c_uint(len(data)), a, out, C.c_ulonglong(cap))
        if r < 0:
            raise RuntimeError(self.lib.zref_last_error().decode(errors="replace"))
        return out.raw[:r]

    def fragment(self, data, fragment=6):
        data = bytes(data)
        cap = len(data) // 64 + 16
        fl = np.zeros(cap, dtype=np.uint32)
        fh = np.zeros(cap, dtype=np.uint32)
        k = self.lib.zref_fragment(data, C.c_ulonglong(len(data)), C.c_int(fragment), fl.ctypes.data_as(C.c_void_p),
                                   fh.ctypes.data_as(C.c_void_p), C.c_ulonglong(cap))
        return fl[:k].copy(), fh[:k].copy()


    def archive_blocks(self, spec, flags):
        """The reference's own `zpaqfranz a` over the tree `spec` (relative path -> bytes), in a child process.
        Returns (date14 of the transaction, number of "d" blocks, the "d" blocks, the "h" blocks)."""
        import subprocess
        import sys
        import tempfile
        code = ("import ctypes as C, sys\n"
                "lib = C.CDLL(%r)\n"
                "a = [x.encode() for x in sys.argv[1:]]\n"
                "arr = (C.c_char_p * len(a))(*a)\n"
                "lib.zref_main.restype = C.c_int\n"
                "sys.exit(lib.zref_main(len(a), arr))\n") % os.path.join(REF_DIR, "libzpaqref.so")
        with tempfile.TemporaryDirectory() as tmp:
            src, archive = os.path.join(tmp, "src"), os.path.join(tmp, "t.zpaq")
            for rel, data in spec.items():
                p = os.path.join(src, rel)
                os.makedirs(os.path.dirname(p), exist_ok=True)
                with open(p, "wb") as f:
                    f.write(data)
            r = subprocess.run([sys.executable, "-c", code, "zpaqfranz", "a", archive, src] + list(flags),
                               capture_output=True, text=True, timeout=900)
            if r.returncode != 0:
                raise RuntimeError(r.stdout[-2000:] + r.stderr[-2000:])
            blocks = split_journal_blocks(open(archive, "rb").read())
        d = b"".join(b for k, _, b in blocks if k == "d")
        h = b"".join(b for k, _, b in blocks if k == "h")
        return blocks[0][1][3:17], sum(1 for k, _, _ in blocks if k == "d"), d, h


ZPAQ_TAG = bytes([0x37, 0x6b, 0x53, 0x74, 0xa0, 0x31, 0x83, 0xd3, 0x8c, 0xb2, 0x28, 0xb0, 0xd3]) + b"zPQ"


def split_journal_blocks(blob):
    """[(kind, name, block bytes)] of a journaling archive: kind is the letter after the 14-digit date."""
    starts = []
    p = blob.find(ZPAQ_TAG)
    while p >= 0:
        starts.append(p)
        p = blob.find(ZPAQ_TAG, p + 16)
    out = []
    for i, s in enumerate(starts):
        e = starts[i + 1] if i + 1 < len(starts) else len(blob)
        b = blob[s:e]
        q = 18
        q += 2 + b[q] + 256 * b[q + 1]
        assert b[q] == 1
        name = b[q + 1: b.index(b"\0", q + 1)].decode()
        assert name.startswith("jDC")
        out.append((name[17], name, b))
    return out


# ---- the reference's answers, recorded ----------------------------------------------------------------------------
# The tests compare with the reference (zpaqfranz's own libzpaq), which is not part of this repository.  Its answers to
# every call the suite makes are stored in tests/golden/ref_answers.json, keyed by a digest of the call (method name and
# arguments, byte strings by SHA-256).  Small results are stored whole; larger ones as length + the first 96 bits of
# their SHA-256, which compare equal to the bytes, text or integer array they stand for.  compressBlock's blocks are always
# stored as digests: the replay regenerates them with the plain-C oracle and hands them out only when their digest is
# the recorded one.  Blocks of several segments, which the tests feed back in and the oracle cannot write, are kept
# whole in tests/golden/ref_blocks.zpaq (back to back, a valid ZPAQ stream; the JSON holds offset and length).
# To record again, with the reference built into oracle/_ref/ and a GPU present:
#     ZQ_REF_RECORD=tests/golden/ref_answers.json python -m pytest tests
ANSWERS = os.path.join(ROOT, "tests", "golden", "ref_answers.json")
_WHOLE = 256             # results up to this many bytes / characters / elements are stored whole
_ALWAYS_WHOLE = ("compress_multi",)     # blocks the tests feed back in and the oracle cannot write (several segments)
_NEVER_WHOLE = ("compress_block",)      # regenerated by the oracle (RecordedRef.compress_block)
_KEY, _DIGEST = 12, 24   # hex digits kept of a call's digest (tells the suite's calls apart) and of a result's SHA-256


def _sha(b):
    import hashlib
    return hashlib.sha256(b).hexdigest()


def _arr_bytes(a):
    return np.ascontiguousarray(np.asarray(a).astype("<i8")).tobytes()


def _norm(x):
    """JSON-able, deterministic form of a call argument."""
    if isinstance(x, (bytes, bytearray, memoryview)):
        return "b:" + _sha(bytes(x))
    if isinstance(x, Digest):
        return x.kind[0] + ":" + x.hex
    if isinstance(x, str) and len(x) > _WHOLE:
        return "s:" + _sha(x.encode())[:_DIGEST]
    if isinstance(x, np.ndarray):
        return "a:" + _sha(_arr_bytes(x))
    if isinstance(x, (list, tuple)):
        return [_norm(v) for v in x]
    if isinstance(x, dict):
        return [[str(k), _norm(x[k])] for k in sorted(x)]
    if isinstance(x, (np.integer, bool)):
        return int(x)
    return x


def _key(name, args, kwargs):
    """Digest of the call, arguments bound to Ref's signature with their defaults (positional or not, same key)."""
    import inspect
    import json
    b = inspect.signature(getattr(Ref, name)).bind(None, *args, **kwargs)
    b.apply_defaults()
    bound = [[k, _norm(v)] for k, v in list(b.arguments.items())[1:]]
    return _sha(json.dumps([name, bound], sort_keys=True).encode())[:_KEY]


class Digest:
    """A recorded result too large to store: equal to the bytes / text / integer array of its length and SHA-256 prefix."""
    __array_ufunc__ = None          # numpy hands `array == Digest` to __eq__ below
    __hash__ = None

    def __init__(self, hexdigest, n, kind):
        self.hex, self.n, self.kind = hexdigest, n, kind      # kind: "bytes", "str" or "array"

    def __len__(self):
        return self.n

    def __eq__(self, other):
        if isinstance(other, Digest):
            return np.bool_(other.hex == self.hex and other.n == self.n)
        if self.kind == "array":
            if np.asarray(other).size != self.n:
                return np.bool_(False)
            b = _arr_bytes(other)
        elif self.kind == "str":
            if not isinstance(other, str) or len(other) != self.n:
                return np.bool_(False)
            b = other.encode()
        else:
            if not isinstance(other, (bytes, bytearray, memoryview)) or len(other) != self.n:
                return np.bool_(False)
            b = bytes(other)
        return np.bool_(_sha(b)[:len(self.hex)] == self.hex)

    def __ne__(self, other):
        return ~self.__eq__(other)

    def __repr__(self):
        return "<reference result: %s of length %d, sha256 %s>" % (self.kind, self.n, self.hex[:16])


def _blocks_path(answers_path):
    return os.path.join(os.path.dirname(answers_path), "ref_blocks.zpaq")


def _encode(v, whole=None):
    """JSON form of a result; whole: True store byte strings whole, False as digests, None by size.
    "b:" base64 bytes, "f:<offset>:<n>" bytes in ref_blocks.zpaq (RecordingRef.save), "h:<digest>:<n>" bytes, "s:" text,
    "H:<digest>:<n>" text (a digest passed back as an argument keys the call as the text would), "A:<digest>:<n>"
    integer array."""
    import base64
    if isinstance(v, Digest):
        return "%s:%s:%d" % ({"bytes": "h", "str": "H", "array": "A"}[v.kind], v.hex, v.n)
    if isinstance(v, (bytes, bytearray)):
        v = bytes(v)
        if whole or (whole is None and len(v) <= _WHOLE):
            return "b:" + base64.b64encode(v).decode()
        return "h:%s:%d" % (_sha(v)[:_DIGEST], len(v))
    if isinstance(v, np.ndarray):
        if v.size <= _WHOLE:
            return {"a": v.tolist(), "dt": v.dtype.str}
        return "A:%s:%d" % (_sha(_arr_bytes(v))[:_DIGEST], v.size)
    if isinstance(v, (list, tuple)):
        return {"t" if isinstance(v, tuple) else "l": [_encode(x, whole) for x in v]}
    if isinstance(v, str):
        return "s:" + v if len(v) <= _WHOLE else "H:%s:%d" % (_sha(v.encode())[:_DIGEST], len(v))
    if isinstance(v, (np.integer, bool)):
        return int(v)
    return v


def _decode(e, blocks):
    import base64
    if isinstance(e, str):
        tag, body = e[0], e[2:]
        if tag == "b":
            return base64.b64decode(body)
        if tag == "s":
            return body
        a, n = body.split(":")
        if tag == "f":
            return blocks[int(a): int(a) + int(n)]
        return Digest(a, int(n), {"h": "bytes", "H": "str", "A": "array"}[tag])
    if not isinstance(e, dict):
        return e
    if "a" in e:
        return np.array(e["a"], dtype=np.dtype(e["dt"]))
    if "t" in e:
        return tuple(_decode(x, blocks) for x in e["t"])
    return [_decode(x, blocks) for x in e["l"]]


def _load_answers(path):
    """(answers, bytes of ref_blocks.zpaq) as stored beside each other."""
    import json
    bp = _blocks_path(path)
    return json.load(open(path)), (open(bp, "rb").read() if os.path.exists(bp) else b"")


class RecordedRef:
    """Ref's interface, answered from tests/golden/ref_answers.json."""

    def __init__(self, answers, blocks, oracle=None):
        self.answers, self.blocks, self.oracle = answers, blocks, oracle

    def __getattr__(self, name):
        if name.startswith("_") or not callable(getattr(Ref, name, None)):
            raise AttributeError(name)

        def call(*args, **kwargs):
            k = _key(name, args, kwargs)
            if k not in self.answers:
                raise KeyError("no recorded reference answer for %s(...): its arguments differ from the recorded call (%s)" % (name, k[:16]))
            return _decode(self.answers[k], self.blocks)
        return call

    def compress_block(self, data, method, filename=None, comment=None, dosha1=True):
        """The recorded block; when only its digest is stored, the oracle's block with that digest."""
        want = self.__getattr__("compress_block")(data, method, filename, comment, dosha1=dosha1)
        if not isinstance(want, Digest) or self.oracle is None:
            return want
        import zpaqfranz_b200 as zq
        data = bytes(data)
        orc = self.oracle
        p = zq.plan_block(method, data)
        a = p["args"]
        d2 = orc.e8e9(data) if a[1] >= 4 else data
        s = orc.lz_stream(d2, a) if (a[1] & 3) else d2
        f = orc.block_modeled if p["header"][6] else orc.block_unmodeled
        cm = ("%d" % len(data) + ("" if comment is None else " " + comment)).encode("latin1")
        fn = None if filename is None else filename.encode("latin1")
        blk = f(p["header"], p["pcomp"], fn, cm, s, orc.sha1(data) if dosha1 else None)
        return blk if want == blk else want     # not the reference's block: only its digest is known


class RecordingRef:
    """The live reference; every answer it gives is kept for RecordedRef."""

    def __init__(self, ref):
        self.ref, self.answers = ref, {}

    def __getattr__(self, name):
        fn = getattr(self.ref, name)
        if name.startswith("_") or not callable(fn):
            return fn

        def call(*args, **kwargs):
            v = fn(*args, **kwargs)
            self.answers[_key(name, args, kwargs)] = _encode(v, True if name in _ALWAYS_WHOLE else False if name in _NEVER_WHOLE else None)
            return v
        return call

    def save(self, path):
        """Merged into the answers already at `path`; whole results over _WHOLE bytes go to ref_blocks.zpaq."""
        import base64
        import json
        answers = {}
        if os.path.exists(path):
            old, blocks = _load_answers(path)
            answers = {k: _encode(_decode(v, blocks), whole=True) for k, v in old.items()}   # digests stay digests
        answers.update(self.answers)
        out = bytearray()
        for k in sorted(answers):
            v = answers[k]
            if isinstance(v, str) and v.startswith("b:"):
                b = base64.b64decode(v[2:])
                if len(b) > _WHOLE:
                    answers[k] = "f:%d:%d" % (len(out), len(b))
                    out += b
        with open(_blocks_path(path), "wb") as f:
            f.write(out)
        with open(path, "w") as f:
            json.dump(answers, f, sort_keys=True, separators=(",", ":"))
            f.write("\n")


def load_oracle():
    return Oracle(C.CDLL(os.path.join(REF_DIR, "libzqoracle.so")))


def load_ref():
    p = os.path.join(REF_DIR, "libzpaqref.so")
    if not os.path.exists(p):
        return None
    return Ref(C.CDLL(p))


def load_recorded_ref(oracle=None):
    return RecordedRef(*_load_answers(ANSWERS), oracle=oracle)
