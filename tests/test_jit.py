"""ZPAQL -> CUDA C translation (zpaqfranz_b200/csrc/zq_jit.cpp): the generated code, compiled for the host, is stepped
against the device interpreter over the same bytes (registers, H, R, M must agree after every byte), and NVRTC compiles
the generated translation unit for sm_90a.  No GPU needed; the compress path does not use the translator yet."""
import ctypes as C
import os
import subprocess

import pytest

import zpaqfranz_b200 as zq
from zpaqfranz_b200 import corpus
from test_cm_emu import CONFIGS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")
CSRC = os.path.join(ROOT, "zpaqfranz_b200", "csrc")

HEADERS = {("method " + m): lambda m=m: bytes(zq.plan_block(m, corpus.text_unit(1, 2000))["header"])
           for m in ["36,200,1", "3", "4", "5", "412,100,0", "56,200,1"]}
HEADERS.update({("config " + n): lambda n=n: bytes(zq.assemble_config(CONFIGS[n])["header"]) for n in sorted(CONFIGS)})
# loops, backward jumps, division, register file, swaps, long jumps
HEADERS["config loops"] = lambda: bytes(zq.assemble_config(
    "comp 4 6 0 0 1 0 cm 12 8 hcomp *c=a c++ b=c a= 0 d= 0 do b-- a+=*b d++ a> 200 if a/= 3 a%= 101 endif d<>a a== 7 d<>a until "
    "r=a 3 a=r 3 a*= 5 *d<>a b<>a c<>a *b<>a d= 0 *d=a a=c a<<= 3 a^=*d a|= 1 a&~ 6 *d=a halt end")["header"])


def _source(header):
    n, err = C.c_uint32(0), C.create_string_buffer(256)
    rc = zq.lib.zq_jit_context_source(header, len(header), None, 0, C.byref(n), err, C.c_size_t(256))
    assert rc == 0, err.value
    buf = C.create_string_buffer(n.value + 1)
    assert zq.lib.zq_jit_context_source(header, len(header), buf, n.value + 1, C.byref(n), err, C.c_size_t(256)) == 0
    return buf.value.decode()


@pytest.mark.parametrize("name", sorted(HEADERS))
def test_translation_matches_interpreter_and_compiles(name, tmp_path):
    header = HEADERS[name]()
    src = _source(header)
    gen = tmp_path / "gen.h"
    gen.write_text(src)
    lib = tmp_path / "libjitcheck.so"
    subprocess.run(["g++", "-O1", "-std=c++17", "-w", "-I" + os.path.join(EMU, "shim"), "-I" + CSRC, "-I" + os.path.join(ROOT, "include"),
                    '-DZQ_JIT_GENERATED="%s"' % gen, "-shared", "-fPIC", "-o", str(lib), os.path.join(EMU, "jit_check.cpp")], check=True)
    chk = C.CDLL(str(lib))
    # HCOMP byte code = header after the component list: hsize(2) hh hm ph pm n comp... 0 hcomp... 0
    hh, hm, n = header[2], header[3], header[6]
    sizes = [0, 2, 3, 2, 3, 4, 6, 6, 3, 5]
    p = 7
    for _ in range(n):
        p += sizes[header[p]]
    code = header[p + 1:]
    for data in (corpus.text_unit(4, 3000), corpus.random_unit(5, 2000), bytes(600), b"abc" * 300 + bytes(range(256))):
        errs = (C.c_int * 2)()
        assert chk.jit_check(code, len(code), hh, hm, data, len(data), errs) == 0, (name, list(errs))
    size, log = C.c_uint32(0), C.create_string_buffer(4096)
    rc = zq.lib.zq_jit_compile(src.encode(), C.byref(size), log, C.c_size_t(4096))
    if rc == zq.ZQ_E_UNSUPPORTED:
        pytest.skip("NVRTC not available: " + log.value.decode())
    assert rc == 0 and size.value > 1000, log.value.decode()


def _raw_header(hcomp, hh=2, hm=4):
    """hsize(2) hh hm ph pm n=0 | 0 | hcomp... (trailing 0 included in hcomp)"""
    body = bytes([hh, hm, 0, 0, 0, 0]) + bytes(hcomp)
    return bytes([len(body) & 255, len(body) >> 8]) + body


@pytest.mark.parametrize("name,hcomp", [
    ("invalid opcode", [1, 5, 56, 0]),                 # a++ ; undefined opcode 5
    ("runs off the end", [1, 9, 0]),                   # no halt: the END marker is executed -> error
    ("jump past the end", [1, 63, 100, 56, 0]),        # jmp +100
    ("jump before the start", [1, 63, 156, 56, 0]),    # jmp -100
    ("error only on some inputs", [219, 65, 39, 2, 56, 0, 5, 56, 0]),   # a== 65 ; jt +2 -> halt... / undefined
])
def test_zpaql_errors_agree(name, hcomp, tmp_path):
    header = _raw_header(hcomp)
    src = _source(header)
    gen = tmp_path / "gen.h"
    gen.write_text(src)
    lib = tmp_path / "libjitcheck.so"
    subprocess.run(["g++", "-O1", "-std=c++17", "-w", "-I" + os.path.join(EMU, "shim"), "-I" + CSRC, "-I" + os.path.join(ROOT, "include"),
                    '-DZQ_JIT_GENERATED="%s"' % gen, "-shared", "-fPIC", "-o", str(lib), os.path.join(EMU, "jit_check.cpp")], check=True)
    chk = C.CDLL(str(lib))
    code = bytes(hcomp)
    for data in (b"AAAA", b"BABA", bytes(range(60, 70))):
        errs = (C.c_int * 2)()
        assert chk.jit_check(code, len(code), 2, 4, data, len(data), errs) == 0, (name, list(errs))


def test_jump_into_an_operand_is_left_to_the_interpreter():
    header = _raw_header([71, 63, 63, 253, 56, 0])     # a= 63 ; jmp -3 lands on the operand byte of "a= 63"
    n, err = C.c_uint32(0), C.create_string_buffer(256)
    assert zq.lib.zq_jit_context_source(header, len(header), None, 0, C.byref(n), err, C.c_size_t(256)) == zq.ZQ_E_UNSUPPORTED
    assert b"middle of an instruction" in err.value


def _coder_source(header):
    n, err = C.c_uint32(0), C.create_string_buffer(256)
    rc = zq.lib.zq_jit_coder_source(header, len(header), None, 0, C.byref(n), err, C.c_size_t(256))
    assert rc == 0, err.value
    buf = C.create_string_buffer(n.value + 1)
    assert zq.lib.zq_jit_coder_source(header, len(header), buf, n.value + 1, C.byref(n), err, C.c_size_t(256)) == 0
    return buf.value.decode()


CODER_MODELS = ["method 36,200,1", "method 3", "method 4", "method 5", "method 412,100,0"] + ["config " + n for n in sorted(CONFIGS)]


@pytest.mark.parametrize("name", CODER_MODELS)
def test_generated_model_codes_like_the_oracle(name, oracle, tmp_path):
    """The model written out as straight-line code (zq_encode_block) + the translated context program, compiled for the
    host: coded bytes equal the oracle's; NVRTC compiles the same translation unit for sm_90a."""
    from test_cm_emu import _coded_by_oracle
    header = HEADERS[name]()
    src = _coder_source(header)
    gen = tmp_path / "gen.h"
    gen.write_text(src)
    lib = tmp_path / "libjitcoder.so"
    subprocess.run(["g++", "-O1", "-std=c++17", "-w", "-I" + CSRC, "-I" + os.path.join(ROOT, "include"), '-DZQ_JIT_GENERATED="%s"' % gen,
                    "-shared", "-fPIC", "-o", str(lib), os.path.join(EMU, "jit_coder_check.cpp"), os.path.join(CSRC, "zq_cm_host.cpp"),
                    os.path.join(CSRC, "zq_config.cpp")], check=True)
    chk = C.CDLL(str(lib))
    chk.jit_encode.restype = C.c_long
    if name.startswith("method "):
        method = name.split(" ", 1)[1]
        datas = [corpus.text_unit(1, 2000), corpus.text_unit(3, 2500), corpus.mixed_unit(5, 2000)]   # the first is the header's own unit
    else:
        method = None
        datas = [b"", b"x", b"abracadabra" * 30, corpus.text_unit(9, 1200), corpus.random_unit(5, 500)]
    ran = 0
    for data in datas:
        if method:
            plan = zq.plan_block(method, data)
            if bytes(plan["header"]) != header:
                continue                                  # another type heuristics outcome -> different model
            pcomp = bytes(plan["pcomp"])
            stream = oracle.lz_stream(data, plan["args"]) if (plan["args"][1] & 3) else data
        else:
            pcomp, stream = b"", data
        payload = (bytes([1, len(pcomp) & 255, len(pcomp) >> 8]) + pcomp) if pcomp else b"\0"
        cap = 2 * len(stream) + 2 * len(payload) + 4096
        out = (C.c_uint8 * cap)()
        r = chk.jit_encode(header, len(header), payload, len(payload), stream, len(stream), out, cap)
        assert r >= 0, r
        assert bytes(out[:r]) == _coded_by_oracle(oracle, header, pcomp, stream), (name, len(data))
        ran += 1
    assert ran > 0
    size, log = C.c_uint32(0), C.create_string_buffer(8192)
    rc = zq.lib.zq_jit_compile(src.encode(), C.byref(size), log, C.c_size_t(8192))
    if rc == zq.ZQ_E_UNSUPPORTED:
        pytest.skip("NVRTC not available: " + log.value.decode())
    assert rc == 0 and size.value > 1000, log.value.decode()


@pytest.mark.parametrize("name,stride", [("method 36,200,1", 32), ("method 3", 1), ("config icm_chain_mix2_sse", 32), ("config four_mixers_big_h", 1)])
def test_generated_kernels_under_the_emulator(name, stride, oracle, tmp_path):
    """zq_ctx_kernel + zq_code_kernel themselves (indexing of the per-group argument arrays, one block per thread or per
    warp, several blocks of different lengths per launch) under the SIMT emulator."""
    import numpy as np
    from test_cm_emu import _coded_by_oracle
    header = HEADERS[name]()
    src = _coder_source(header)
    gen = tmp_path / "gen.h"
    gen.write_text(src)
    lib = tmp_path / "libjitkernels.so"
    subprocess.run(["g++", "-O1", "-std=c++17", "-w", "-I" + os.path.join(EMU, "shim"), "-I" + CSRC, "-I" + os.path.join(ROOT, "include"),
                    '-DZQ_JIT_GENERATED="%s"' % gen, "-shared", "-fPIC", "-o", str(lib), os.path.join(EMU, "jit_kernel_check.cpp"),
                    os.path.join(CSRC, "zq_cm_host.cpp"), os.path.join(CSRC, "zq_config.cpp")], check=True)
    chk = C.CDLL(str(lib))
    if name.startswith("method "):
        method = name.split(" ", 1)[1]
        datas = [corpus.text_unit(1, 2000), corpus.text_unit(1, 2000)[:700], corpus.text_unit(3, 1500), corpus.text_unit(4, 40), corpus.text_unit(5, 1100)]
        streams, pcomp = [], b""
        for d in datas:
            plan = zq.plan_block(method, d)
            if bytes(plan["header"]) != header:
                continue
            pcomp = bytes(plan["pcomp"])
            streams.append(oracle.lz_stream(d, plan["args"]) if (plan["args"][1] & 3) else d)
    else:
        pcomp = b""
        streams = [b"abracadabra" * 30, b"", corpus.text_unit(9, 900), b"x", corpus.random_unit(5, 400)]
    assert len(streams) >= 3
    payload = (bytes([1, len(pcomp) & 255, len(pcomp) >> 8]) + pcomp) if pcomp else b"\0"
    blob = b"".join(streams) + b"\0" * 16
    slen = np.array([len(s) for s in streams], dtype=np.uint32)
    soff = np.concatenate([[0], np.cumsum(slen.astype(np.uint64))[:-1]]).astype(np.uint64)
    cap = 2 * int(slen.max()) + 2 * len(payload) + 4096
    out = (C.c_uint8 * (cap * len(streams)))()
    olen = (C.c_uint32 * len(streams))()
    rc = chk.jit_kernels(header, len(header), payload, len(payload), blob, soff.ctypes.data_as(C.c_void_p), slen.ctypes.data_as(C.c_void_p),
                         len(streams), stride, out, cap, olen)
    assert rc == 0
    raw = bytes(out)
    for t, s in enumerate(streams):
        assert raw[t * cap: t * cap + olen[t]] == _coded_by_oracle(oracle, header, pcomp, s), (name, t, len(s))
