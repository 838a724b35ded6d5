#!/usr/bin/env python3
"""Extract the reference's X448 vectors into tests/golden/x448.json (data only; the JSON is committed and the tests
read nothing else).

    python tools/extract_x448_golden.py <path to a RustCrypto/elliptic-curves checkout>

Sources (relative to the checkout):
  x448/src/lib.rs  test_rfc_test_vectors_fixed        RFC 7748 section 5.2, the two single-shot vectors
  x448/src/lib.rs  test_rfc_test_vectors_alice_bob    RFC 7748 section 6.2, secrets, public keys and the shared secret
  x448/src/lib.rs  test_rfc_test_vectors_iteration    RFC 7748 section 5.2, the 1 / 1,000 / 1,000,000 iteration values
  ed448-goldilocks/src/montgomery.rs  MontgomeryPoint::LOW_A / LOW_B / LOW_C (the encodings x448::x448 refuses)
"""
import json
import os
import re
import sys

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "x448.json")
ARRAY = r"\[((?:\s*0x[0-9a-fA-F]+\s*,?)+)\s*\]"


def hexbytes(body):
    b = bytes(int(t, 16) for t in re.findall(r"0x([0-9a-fA-F]+)", body))
    assert len(b) == 56, len(b)
    return b.hex()


def fn_body(text, name):
    i = text.index(f"fn {name}(")
    j = text.find("\n    #[test]", i)
    return text[i:j if j > 0 else len(text)]


def main():
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    ref = sys.argv[1]
    lib = open(os.path.join(ref, "x448", "src", "lib.rs")).read()
    mont = open(os.path.join(ref, "ed448-goldilocks", "src", "montgomery.rs")).read()

    fixed = fn_body(lib, "test_rfc_test_vectors_fixed")
    secrets = [hexbytes(m) for m in re.findall(r"secret:\s*" + ARRAY, fixed)]
    points = [hexbytes(m) for m in re.findall(r"point:\s*" + ARRAY, fixed)]
    expected = [hexbytes(m) for m in re.findall(r"expected:\s*" + ARRAY, fixed)]
    assert len(secrets) == len(points) == len(expected) == 2

    ab = fn_body(lib, "test_rfc_test_vectors_alice_bob")
    privs = [hexbytes(m) for m in re.findall(r"EphemeralSecret::from\(" + ARRAY + r"\)", ab)]
    named = {n: hexbytes(m) for n, m in re.findall(r"let (\w+) = " + ARRAY, ab)}
    assert len(privs) == 2

    it = fn_body(lib, "test_rfc_test_vectors_iteration")
    iters = {n: hexbytes(m) for n, m in re.findall(r"let (\w+) = " + ARRAY, it)}

    low = {n: hexbytes(m) for n, m in re.findall(r"pub const (LOW_[ABC]): MontgomeryPoint = MontgomeryPoint\(" + ARRAY + r"\)", mont)}
    assert sorted(low) == ["LOW_A", "LOW_B", "LOW_C"]

    data = {
        "source": "x448/src/lib.rs tests (RFC 7748 sections 5.2 and 6.2), ed448-goldilocks/src/montgomery.rs LOW_*",
        "fixed": [{"k": k, "u": u, "out": o} for k, u, o in zip(secrets, points, expected)],
        "alice_bob": {"alice_priv": privs[0], "alice_pub": named["expected_alice_pub"], "bob_priv": privs[1],
                      "bob_pub": named["expected_bob_pub"], "shared": named["expected_shared"]},
        "iterations": {"1": iters["one_iter"], "1000": iters["one_k_iter"], "1000000": iters["one_mil_iter"]},
        "low_order": low,
    }
    with open(OUT, "w") as f:
        json.dump(data, f, indent=1)
        f.write("\n")
    print("wrote", os.path.normpath(OUT))


if __name__ == "__main__":
    main()
