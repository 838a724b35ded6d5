#!/usr/bin/env python3
"""Extract the reference's Ed448 vectors into tests/golden/ed448.json (data only; the JSON is committed and the tests
read nothing else).

    python tools/extract_ed448_golden.py <path to a RustCrypto/elliptic-curves checkout>

Sources (relative to the checkout):
  ed448-goldilocks/src/sign/verifying_key.rs  TEST_VECTORS   RFC 8032 section 7.4 / 7.5: seed, public key, message,
                                                             Ed448ph flag, context and signature of the six vectors;
                                              fn signatures  the negative cases it checks for each vector
  ed448-goldilocks/src/edwards/affine.rs      CompressedEdwardsY::GENERATOR   the compressed base point
  ed448-goldilocks/src/field/scalar.rs        ORDER          the group order ell
"""
import json
import os
import re
import sys

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "ed448.json")


def main():
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    ref = os.path.join(sys.argv[1], "ed448-goldilocks", "src")
    vk = open(os.path.join(ref, "sign", "verifying_key.rs")).read()
    affine = open(os.path.join(ref, "edwards", "affine.rs")).read()
    scalar = open(os.path.join(ref, "field", "scalar.rs")).read()

    body = vk[vk.index("const TEST_VECTORS"):vk.index("fn signatures()")]
    vectors = []
    for blk in re.findall(r"Ed448TestVector\s*\{(.*?)\}", body, re.S):
        f = dict(re.findall(r'(\w+):\s*"([0-9a-fA-F]*)"', blk))
        ph = re.search(r"ph:\s*(true|false)", blk).group(1) == "true"
        vectors.append({"seed": f["s"], "public": f["q"], "msg": f["m"], "prehashed": ph, "ctx": f["ctx"], "sig": f["sig"]})
    assert len(vectors) == 6, len(vectors)

    # the negative cases of fn signatures(): another context [1], message [0] (Ed448), byte 42 of PH(M) ^ 0x08 (Ed448ph)
    test = vk[vk.index("fn signatures()"):]
    assert "&[1u8]" in test and "&[0u8]" in test and "hm[42] ^= 0x08" in test
    negatives = {"wrong_context": "01", "wrong_message": "00", "prehash_flip": {"byte": 42, "xor": 8}}

    g = re.search(r"pub const GENERATOR: Self = Self\(\[(.*?)\]\)", affine, re.S).group(1)
    gen = bytes(int(t) for t in re.findall(r"\d+", g))
    assert len(gen) == 57

    order = re.search(r'pub const ORDER: Odd<U448> = Odd::<U448>::from_be_hex\(\s*"([0-9a-f]+)"', scalar).group(1)

    data = {
        "source": "ed448-goldilocks/src/sign/verifying_key.rs TEST_VECTORS and fn signatures (RFC 8032 section 7.4-7.5), "
                  "edwards/affine.rs CompressedEdwardsY::GENERATOR, field/scalar.rs ORDER",
        "vectors": vectors,
        "negatives": negatives,
        "generator": gen.hex(),
        "order": order,
    }
    with open(OUT, "w") as f:
        json.dump(data, f, indent=1)
        f.write("\n")
    print("wrote", os.path.normpath(OUT))


if __name__ == "__main__":
    main()
