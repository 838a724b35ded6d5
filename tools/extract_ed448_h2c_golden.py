#!/usr/bin/env python3
"""Extract the reference's Ed448 hash-to-curve vectors into tests/golden/ed448_h2c.json (data only; the JSON is committed
and the tests read nothing else).

    python tools/extract_ed448_h2c_golden.py <path to a RustCrypto/elliptic-curves checkout>

Sources (relative to the checkout):
  ed448-goldilocks/src/edwards/extended.rs  fn hash_with_test_vectors  RFC 9380 edwards448_XOF:SHAKE256_ELL2_RO_: DST, and
                                                                       per message the affine (x, y) of hash_from_bytes
                                            fn encode                  the same for _NU_ (encode_from_bytes)
  ed448-goldilocks/src/field/element.rs     fn from_okm_curve448       hash_to_field's u0, u1 under the curve448 RO DST
                                            fn from_okm_edwards448     the same under the edwards448 RO DST
  ed448-goldilocks/src/edwards/scalar.rs    fn scalar_hash             one hash_to_scalar::<Ed448, _, U84> vector
Coordinates and field elements are kept as the reference writes them: big-endian hex.
"""
import json
import os
import re
import sys

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "ed448_h2c.json")


def rust_bytes(s: str) -> bytes:
    """a Rust byte-string literal b"..." body with \\xNN escapes"""
    return re.sub(r"\\x([0-9a-fA-F]{2})", lambda m: chr(int(m.group(1), 16)), s).encode("latin-1")


def between(text: str, start: str, end: str) -> str:
    i = text.index(start)
    return text[i:text.index(end, i)]


def triples(body: str, keys):
    """the (b"msg", hex!("..."), hex!("...")) entries of a test table and its DST"""
    dst = rust_bytes(re.search(r'const DST: &\[u8\] = b"(.*?)";', body).group(1))
    rows = re.findall(r'\(b"(.*?)",\s*hex!\("([0-9a-f]+)"\),\s*hex!\("([0-9a-f]+)"\)\)', body)
    assert len(rows) == 5 and all(len(a) == 112 and len(b) == 112 for _, a, b in rows), rows
    return {"dst": dst.hex(), "vectors": [{"msg": rust_bytes(m).hex(), keys[0]: a, keys[1]: b} for m, a, b in rows]}


def main():
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    src = os.path.join(sys.argv[1], "ed448-goldilocks", "src")
    extended = open(os.path.join(src, "edwards", "extended.rs")).read()
    element = open(os.path.join(src, "field", "element.rs")).read()
    scalar = open(os.path.join(src, "edwards", "scalar.rs")).read()

    ro = triples(between(extended, "fn hash_with_test_vectors", "fn hash_fuzzing"), ("x", "y"))
    nu = triples(between(extended, "fn encode()", "assert_eq!(p.y.to_bytes(), yy);"), ("x", "y"))
    okm_c = triples(between(element, "fn from_okm_curve448", "assert_from_okm"), ("u0", "u1"))
    okm_e = triples(between(element, "fn from_okm_edwards448", "assert_from_okm"), ("u0", "u1"))

    sh = between(scalar, "fn scalar_hash", "assert_eq!")
    scalar_hash = {
        "msg": rust_bytes(re.search(r'let msg = b"(.*?)";', sh).group(1)).hex(),
        "dst": rust_bytes(re.search(r'let dst = b"(.*?)";', sh).group(1)).hex(),
        "scalar": re.search(r'hex!\(\s*"([0-9a-f]+)"', sh).group(1),
    }
    assert len(scalar_hash["scalar"]) == 114

    data = {
        "source": "ed448-goldilocks/src/edwards/extended.rs hash_with_test_vectors (RO) and encode (NU); field/element.rs "
                  "from_okm_curve448 and from_okm_edwards448 (hash_to_field); edwards/scalar.rs scalar_hash. "
                  "Coordinates and field elements big-endian hex, as the reference writes them.",
        "hash_to_curve": ro,
        "encode_to_curve": nu,
        "from_okm_curve448": okm_c,
        "from_okm_edwards448": okm_e,
        "scalar_hash": scalar_hash,
    }
    with open(OUT, "w") as f:
        json.dump(data, f, indent=1)
        f.write("\n")
    print("wrote", os.path.normpath(OUT))


if __name__ == "__main__":
    main()
