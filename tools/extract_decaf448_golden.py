#!/usr/bin/env python3
"""Extract the reference's Decaf448 vectors into tests/golden/decaf448.json (data only; the JSON is committed and the
tests read nothing else).

    python tools/extract_decaf448_golden.py <path to a RustCrypto/elliptic-curves checkout>

Sources (relative to the checkout):
  ed448-goldilocks/src/decaf.rs         fn hash_to_curve           RFC 9496 "group elements from uniform byte strings":
                                                                   112 uniform bytes and DecafPoint::from_uniform_bytes
  ed448-goldilocks/src/decaf/points.rs  fn test_vectors_lib_decaf  the encodings of [k]G for k = 0..15 (libdecaf)
                                        fn test_invalid_point      two records decompress refuses
                                        CompressedDecaf::GENERATOR the encoding of G
  ed448-goldilocks/src/decaf/scalar.rs  fn scalar_hash             one hash_to_scalar vector (message, DST, scalar)
                                        fn hash_to_scalar_voprf    RFC 9497 decaf448-SHAKE256 DeriveKeyPair: seed,
                                                                   key info, the three DSTs and their secret scalars
"""
import json
import os
import re
import sys

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "decaf448.json")


def rust_bytes(s: str) -> bytes:
    """a Rust byte-string literal b"..." body with \\xNN escapes"""
    return re.sub(r"\\x([0-9a-fA-F]{2})", lambda m: chr(int(m.group(1), 16)), s).encode("latin-1")


def main():
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    ref = os.path.join(sys.argv[1], "ed448-goldilocks", "src", "decaf")
    decaf_rs = open(os.path.join(sys.argv[1], "ed448-goldilocks", "src", "decaf.rs")).read()
    points = open(os.path.join(ref, "points.rs")).read()
    scalar = open(os.path.join(ref, "scalar.rs")).read()

    body = points[points.index("fn test_vectors_lib_decaf"):points.index("fn test_invalid_point")]
    multiples = []
    for blk in re.findall(r"CompressedDecaf\(\[(.*?)\]\)", body, re.S):
        b = bytes(int(t) for t in re.findall(r"\d+", blk))
        assert len(b) == 56
        multiples.append(b.hex())
    assert len(multiples) == 16, len(multiples)

    inv = points[points.index("fn test_invalid_point"):points.index("fn test_hash_to_curve")]
    invalid = [bytes([int(v)] * int(n)).hex() for v, n in re.findall(r"CompressedDecaf\(\[(\d+)u8;\s*(\d+)\]\)", inv)]
    assert len(invalid) == 2, invalid

    g = re.search(r"pub const GENERATOR: Self = Self\(\[(.*?)\]\)", points, re.S).group(1)
    gen = bytes(int(t) for t in re.findall(r"\d+", g))
    assert len(gen) == 56 and gen.hex() == multiples[1]

    sh = scalar[scalar.index("fn scalar_hash"):scalar.index("fn hash_to_scalar_voprf")]
    scalar_hash = {
        "msg": rust_bytes(re.search(r'let msg = b"(.*?)";', sh).group(1)).hex(),
        "dst": rust_bytes(re.search(r'let dst = b"(.*?)";', sh).group(1)).hex(),
        "scalar": re.search(r'hex!\(\s*"([0-9a-f]+)"', sh).group(1),
    }

    vo = scalar[scalar.index("fn hash_to_scalar_voprf"):]
    key_info = rust_bytes(re.search(r'const KEY_INFO: &\[u8\] = b"(.*?)";', vo).group(1))
    seed = re.search(r'const SEED: &\[u8\] =\s*&hex!\("([0-9a-f]+)"\)', vo).group(1)
    derive = []
    for dst, sk in re.findall(r'dst: b"(.*?)",\s*sk_sm: &hex!\(\s*"([0-9a-f]+)"', vo, re.S):
        derive.append({"dst": rust_bytes(dst).hex(), "sk": sk})
    assert len(derive) == 3, derive

    uniform = [{"input": i, "output": o}
               for i, o in re.findall(r'input: hex!\(\s*"([0-9a-f]+)"\s*\),\s*output: hex!\(\s*"([0-9a-f]+)"\s*\)', decaf_rs)]
    assert len(uniform) == 7 and all(len(u["input"]) == 224 and len(u["output"]) == 112 for u in uniform), uniform

    data = {
        "source": "ed448-goldilocks/src/decaf.rs hash_to_curve (RFC 9496 uniform-bytes vectors); decaf/points.rs test_vectors_lib_decaf, test_invalid_point, CompressedDecaf::GENERATOR; "
                  "decaf/scalar.rs scalar_hash and hash_to_scalar_voprf (RFC 9497 decaf448-SHAKE256 DeriveKeyPair)",
        "generator": gen.hex(),
        "multiples": multiples,
        "from_uniform_bytes": uniform,
        "invalid": invalid,
        "scalar_hash": scalar_hash,
        "derive_key_pair": {"seed": seed, "info": key_info.hex(), "vectors": derive},
    }
    with open(OUT, "w") as f:
        json.dump(data, f, indent=1)
        f.write("\n")
    print("wrote", os.path.normpath(OUT))


if __name__ == "__main__":
    main()
