"""Committed golden vectors (tests/golden/blocks.json, produced by the reference through
tests/golden/make_golden.py): the plain-C oracle on CPU, and the CUDA path on the GPU, must reproduce
them byte for byte even where the reference itself is not available."""
import base64
import json
import os

import numpy as np
import pytest

G = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "blocks.json")))
INPUTS = {k: base64.b64decode(v) for k, v in G["inputs"].items()}


def test_oracle_reproduces_golden_blocks(zq, oracle):
    for e in G["blocks"]:
        d, m = INPUTS[e["input"]], e["method"]
        p = zq.plan_block(m, d)
        a = p["args"]
        if a[1] >= 4:
            d2 = oracle.e8e9(d)
        else:
            d2 = d
        s = oracle.lz_stream(d2, a) if (a[1] & 3) else d2
        f = oracle.block_modeled if p["header"][6] else oracle.block_unmodeled
        blk = f(p["header"], p["pcomp"], b"file", ("%d jDC\x01" % len(d)).encode(), s, oracle.sha1(d))
        assert blk == base64.b64decode(e["block"]), (e["input"], m)


def test_oracle_sha1_matches_golden_digests(oracle):
    for k, d in INPUTS.items():
        assert oracle.sha1(d).hex() == G["digests"][k]["sha1"]


@pytest.mark.gpu
def test_gpu_reproduces_golden_blocks_and_digests(ctx):
    names = list(INPUTS)
    lens = np.array([len(INPUTS[k]) for k in names], dtype=np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens.astype(np.uint64))[:-1]]).astype(np.uint64)
    arena = np.frombuffer(b"".join(INPUTS[k] for k in names) + b"\0", dtype=np.uint8)
    methods = sorted({e["method"] for e in G["blocks"]})
    want = {(e["input"], e["method"]): base64.b64decode(e["block"]) for e in G["blocks"]}
    for m in methods:
        out, ooff, olen = ctx.compress_blocks(arena.copy(), offs, lens, method=m, filename="file", comment="jDC\x01")
        for i, k in enumerate(names):
            assert out[int(ooff[i]): int(ooff[i]) + int(olen[i])].tobytes() == want[(k, m)], (k, m)
    for algo in ("sha1", "sha256", "xxh3_128", "blake3"):
        got = getattr(ctx, algo)(arena, offs, lens)
        for i, k in enumerate(names):
            assert got[i].tobytes().hex() == G["digests"][k][algo], (algo, k)
