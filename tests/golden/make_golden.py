"""Generates tests/golden/blocks.json from the REFERENCE itself (oracle/_ref/libzpaqref.so, built from
the reference's zpaqfranz.cpp by oracle/Makefile): for small deterministic inputs and a spread of methods, the exact
bytes libzpaq::compressBlock writes, plus reference digests.  Run where oracle/_ref/libzpaqref.so is built:
    python tests/golden/make_golden.py
The fixtures let the parity tests run where neither the reference nor the prebuilt _ref exists."""
import base64
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_bindings as ob  # noqa: E402
from zpaqfranz_b200 import corpus  # noqa: E402

INPUTS = {
    "empty": b"", "a": b"a", "abc10": b"abcabcabcabcabc" * 10, "zeros3000": bytes(3000),
    "text6000": corpus.text_unit(1, 6000), "random1500": corpus.random_unit(2, 1500), "repeats5000": corpus.repeats_unit(3, 5000),
}
METHODS = ["0", "1", "2", "3", "36,200,1", "4", "46,200,1", "5", "1,128,2", "x0,0c0,0,255i2,13m8,24s", "x0,2,12,0,7,21,1c0,0,511i2"]


def main():
    ref = ob.load_ref()
    out = {"inputs": {k: base64.b64encode(v).decode() for k, v in INPUTS.items()}, "blocks": [], "digests": {}}
    for name, data in INPUTS.items():
        for m in METHODS:
            blk = ref.compress_block(data, m, "file", "jDC\x01")
            out["blocks"].append({"input": name, "method": m, "block": base64.b64encode(blk).decode()})
        out["digests"][name] = {"sha1": ref.sha1(data).hex(), "sha256": ref.sha256(data).hex(), "xxh3_128": ref.xxh3_128(data).hex(),
                                "blake3": ref.blake3(data).hex()}
    json.dump(out, open(os.path.join(HERE, "blocks.json"), "w"), indent=0)
    print("wrote", len(out["blocks"]), "blocks")


if __name__ == "__main__":
    main()
