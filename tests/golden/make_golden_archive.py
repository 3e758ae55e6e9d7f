"""Generates tests/golden/sha256_zpaq.json: what the REFERENCE's own decoder (oracle/_ref) makes of every block of the
decoder fixture the reference ships, AUTOTEST/sha256.zpaq (copied verbatim to tests/golden/sha256.zpaq; -m5, 256 files
of 37 000 bytes named by the SHA-256 of their content, AUTOTEST/README.txt:1-45).  Run where oracle/_ref/libzpaqref.so is built:
    python tests/golden/make_golden_archive.py"""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_bindings as ob  # noqa: E402

TAG = bytes([0x37, 0x6b, 0x53, 0x74, 0xa0, 0x31, 0x83, 0xd3, 0x8c, 0xb2, 0x28, 0xb0, 0xd3])
PREFIX = 150000     # bytes of the 9.47 MB data block the device test decodes (one warp owns a block)


def split_blocks(a):
    offs, i = [], a.find(TAG)
    while i >= 0:
        offs.append(i)
        i = a.find(TAG, i + 1)
    return [(o, (offs[k + 1] if k + 1 < len(offs) else len(a)) - o) for k, o in enumerate(offs)]


def main():
    ref = ob.load_ref()
    a = open(os.path.join(HERE, "sha256.zpaq"), "rb").read()
    assert hashlib.sha256(a).hexdigest().upper() == "D90223FAEE2878D7854B9438864B4856A3C1F920C34EFB8C136A8949B54E5400"   # README.txt:43
    out = {"archive_sha256": hashlib.sha256(a).hexdigest(), "prefix": PREFIX, "blocks": []}
    for off, ln in split_blocks(a):
        dec = ref.decompress(a[off:off + ln], 64 << 20)
        out["blocks"].append({"offset": off, "length": ln, "decoded_len": len(dec), "sha256": hashlib.sha256(dec).hexdigest(),
                              "prefix_sha256": hashlib.sha256(dec[:PREFIX]).hexdigest()})
    json.dump(out, open(os.path.join(HERE, "sha256_zpaq.json"), "w"), indent=1)
    print("wrote", len(out["blocks"]), "blocks")


if __name__ == "__main__":
    main()
