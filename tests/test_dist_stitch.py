"""One stream cut across the ranks (zq_dist_stitch_fragments, zpaqfranz_b200/csrc/zq_dist.cpp): every rank fragments its
piece speculatively, the collective decides which fragments are the stream's real ones.  The result must be the
fragment list the reference's single sequential chunker (Z:122457-122561) cuts from the whole stream.

CPU tests: the ranks are threads of this process, the all-gather a barrier; the pieces are fragmented by the oracle.
GPU test: the same protocol with every piece fragmented (and hashed) by the device fragmenter."""
import hashlib
import threading

import numpy as np
import pytest

import zpaqfranz_b200 as zq
from zpaqfranz_b200 import corpus


class _ThreadGather:
    """all-gather among `world` threads of one process"""

    def __init__(self, world):
        self.world = world
        self.slots = [b""] * world
        self.bar = threading.Barrier(world)

    def fn(self, rank):
        def ag(data):
            self.slots[rank] = bytes(data)
            self.bar.wait(timeout=120)
            out = list(self.slots)
            self.bar.wait(timeout=120)
            return out
        return ag


def _run_ranks(world, data, fragment, overlap, frag_fn):
    """frag_fn(piece_bytes) -> (lengths, digests or None).  Returns per-rank (lens, digests, record, rounds)."""
    total = len(data)
    tg = _ThreadGather(world)
    res = [None] * world
    err = []

    def work(rank):
        try:
            d = zq.Dist(-1, rank, world, allgather=tg.fn(rank))
            lo, hi = zq.shard_range(total, rank, world)
            avail = min(total, hi + overlap) if rank < world - 1 else total
            start, rounds = lo, 0
            while True:
                lens, dig = frag_fn(data[start:avail])
                while True:
                    st = d.stitch_fragments(total, lo, hi, start, avail, lens)
                    rounds += 1
                    if not st["again"] or st["restart"]:
                        break
                if not st["again"]:
                    break
                start = st["restart_at"]
                assert lo <= start <= avail
            k0, k1 = st["first_keep"], st["first_keep"] + st["n_keep"]
            res[rank] = (np.asarray(lens[k0:k1]), None if dig is None else np.asarray(dig[k0:k1]), st, rounds, d.bytes_exchanged())
            d.close()
        except Exception as e:   # noqa: BLE001
            err.append((rank, repr(e)))
            try:
                tg.bar.abort()
            except Exception:   # noqa: BLE001
                pass

    ts = [threading.Thread(target=work, args=(r,)) for r in range(world)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=600)
    assert not err, err
    return res


def _check(res, data, want_lens):
    got = np.concatenate([r[0] for r in res])
    assert got.tolist() == list(want_lens)
    at = 0
    for r in res:                                   # records are consistent: contiguous byte ranges and fragment numbers
        st = r[2]
        assert st["global_total"] == len(want_lens)
        assert st["global_first"] == at and st["begin"] == int(np.sum(want_lens[:at]))
        at += st["n_keep"]
        assert st["end"] == int(np.sum(want_lens[:at]))
    assert at == len(want_lens)


def _stream(kind, n):
    if kind == "text":
        return corpus.text_bytes(41, n).tobytes()
    if kind == "mixed":
        parts, k = [], 0
        while sum(map(len, parts)) < n:
            parts.append(corpus.mixed_unit(100 + k, 40000 + 7919 * (k % 5)))
            k += 1
        return b"".join(parts)[:n]
    if kind == "zeros_at_cut":                     # a constant run across the cut: the chains never meet by themselves
        return corpus.text_bytes(7, n // 4).tobytes() + bytes(n // 2) + corpus.text_bytes(8, n - n // 4 - n // 2).tobytes()
    raise ValueError(kind)


@pytest.mark.parametrize("world", [2, 3, 4])
@pytest.mark.parametrize("kind", ["text", "mixed", "zeros_at_cut"])
def test_stitched_pieces_equal_the_whole_stream(oracle, world, kind):
    fragment = 1                                   # fragments of 128 .. 16256 bytes: many boundaries in a small stream
    data = _stream(kind, 900_000)
    want, _ = oracle.fragment(data, fragment)
    res = _run_ranks(world, data, fragment, overlap=3 * (8128 << fragment), frag_fn=lambda p: (oracle.fragment(p, fragment)[0], None))
    _check(res, data, want.tolist())
    if kind == "zeros_at_cut":
        assert max(r[3] for r in res) > 1          # the restart path was taken: not a vacuous case
    else:
        assert all(r[3] == 1 for r in res)         # ordinary data: the chains meet inside the overlap, one round
    assert all(r[4] > 0 for r in res)


@pytest.mark.parametrize("total,world", [(0, 2), (1, 3), (5, 4), (300, 4), (5000, 3)])
def test_streams_shorter_than_the_cut(oracle, total, world):
    """pieces that are empty or end before their first boundary: the whole stream is the left ranks' fragments"""
    data = corpus.text_bytes(9, max(total, 1)).tobytes()[:total]
    want = oracle.fragment(data, 1)[0].tolist() if total else []
    res = _run_ranks(world, data, 1, overlap=3 * (8128 << 1),
                     frag_fn=lambda p: (oracle.fragment(p, 1)[0] if len(p) else np.zeros(0, np.uint32), None))
    assert np.concatenate([r[0] for r in res]).tolist() == want
    assert all(r[2]["global_total"] == len(want) for r in res)


def test_overlap_shorter_than_a_fragment_is_refused(oracle):
    data = corpus.text_bytes(5, 400_000).tobytes()  # no overlap at all: the left piece holds no boundary past its end
    tg = _ThreadGather(2)
    out = [None, None]

    def work(rank):
        d = zq.Dist(-1, rank, 2, allgather=tg.fn(rank))
        lo, hi = zq.shard_range(len(data), rank, 2)
        avail = hi if rank == 0 else len(data)
        lens, _ = oracle.fragment(data[lo:avail], 1)
        try:
            d.stitch_fragments(len(data), lo, hi, lo, avail, lens)
            out[rank] = "ok"
        except zq.ZqError as e:
            out[rank] = e.code
        d.close()

    ts = [threading.Thread(target=work, args=(r,)) for r in range(2)]
    [t.start() for t in ts]
    [t.join(timeout=120) for t in ts]
    assert out == [zq.ZQ_E_UNSUPPORTED, zq.ZQ_E_UNSUPPORTED]


def test_single_rank_keeps_everything(oracle):
    data = corpus.text_bytes(3, 200_000).tobytes()
    lens, _ = oracle.fragment(data, 2)
    d = zq.Dist(-1, 0, 1)
    st = d.stitch_fragments(len(data), 0, len(data), 0, len(data), lens)
    assert (st["first_keep"], st["n_keep"], st["global_first"], st["global_total"], st["begin"], st["end"], st["again"]) == \
        (0, len(lens), 0, len(lens), 0, len(data), 0)
    with pytest.raises(zq.ZqError):
        d.stitch_fragments(len(data), 0, len(data), 0, len(data), lens[:-1])      # lengths must add up to the piece
    d.close()


def test_cpp_caller_of_the_c_abi(zq, oracle, tmp_path):
    """tests/cpp/stitch_driver.cpp: the same protocol written as the archiver's host code would (C++ threads as ranks,
    zq_dist_create_cb, zq_dist_stitch_fragments through the C ABI, the checker's chunker linked in)."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = tmp_path / "stitch_driver"
    subprocess.run(["g++", "-O1", "-std=c++17", "-pthread", "-I" + os.path.join(root, "include"), os.path.join(root, "tests/cpp/stitch_driver.cpp"),
                    "-o", str(exe), "-L" + os.path.join(root, "zpaqfranz_b200"), "-lzqb200", "-L" + os.path.join(root, "oracle", "_ref"), "-lzqoracle",
                    "-Wl,-rpath," + os.path.join(root, "zpaqfranz_b200"), "-Wl,-rpath," + os.path.join(root, "oracle", "_ref")], check=True)
    for world, kind in ((2, 0), (3, 0), (4, 1)):
        r = subprocess.run([str(exe), str(world), str(kind)], capture_output=True, text=True, timeout=120)
        assert r.returncode == 0 and r.stdout.startswith("OK"), r.stdout + r.stderr
        if kind == 1:
            assert "1 call(s)" not in r.stdout          # the restart path was taken


@pytest.mark.gpu
@pytest.mark.parametrize("kind,world", [("mixed", 3), ("zeros_at_cut", 2)])
def test_device_fragmenter_pieces_equal_the_whole_stream(ctx, oracle, kind, world):
    """Every piece through zq_fragment on the GPU (fragment 6, the archiver's default): lengths and SHA-1s of the
    kept fragments equal those of one zq_fragment call over the whole stream and the oracle's lengths."""
    fragment = 6
    data = _stream(kind, 24_000_000)
    arr = np.frombuffer(data, dtype=np.uint8)
    wl, _, wsha, _ = ctx.fragment(arr, [0], [len(data)], fragment=fragment)
    assert wl.tolist() == oracle.fragment(data, fragment)[0].tolist()
    lock = threading.Lock()                        # one context: the ranks take turns on the device

    def frag(piece):
        p = np.frombuffer(piece, dtype=np.uint8)
        if len(p) == 0:
            return np.zeros(0, np.uint32), np.zeros((0, 20), np.uint8)
        with lock:
            fl, _, fs, _ = ctx.fragment(p, [0], [len(p)], fragment=fragment)
        return fl, fs

    res = _run_ranks(world, data, fragment, overlap=4 * (8128 << fragment), frag_fn=frag)
    _check(res, data, wl.tolist())
    got_sha = np.concatenate([r[1] for r in res])
    assert (got_sha == wsha).all()
    at = 0
    for k in (0, len(wl) // 2, len(wl) - 1):       # and they are the SHA-1s of those bytes
        at = int(wl[:k].sum())
        assert bytes(got_sha[k]) == hashlib.sha1(data[at:at + int(wl[k])]).digest()
