"""ECG_INLINE_LOOPS=0 keeps the call-based field operations in the fixed-base and bucket-accumulation kernels of secp256k1
and P-256 (ecgpu.cu: inline_loops).  The setting is read once per process, so each configuration runs in its own
interpreter; both must give the same bytes."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = r"""
import sys, random
import numpy as np
for p in sys.argv[2:]:
    sys.path.insert(0, p)
import ecgpu, pyref
from helpers import pack_points, pack_scalars, edge_scalars
eng = ecgpu.Engine([0])
out = {}
for curve in ("k256", "p256"):
    c = pyref.CURVES[curve]
    rng = random.Random(7)
    ks = edge_scalars(c) + [rng.randrange(c.n) for _ in range(3000)]
    xy, inf = eng.mul_by_generator(curve, pack_scalars(ks))
    out[curve + "_kg_xy"], out[curve + "_kg_inf"] = np.asarray(xy), np.asarray(inf)
    n = 1 << 13  # the bucket method's threshold
    base = [pyref.mul(c, rng.randrange(1, c.n), pyref.G(c)) for _ in range(64)]
    Ps = [base[rng.randrange(64)] for _ in range(n)]
    pxy, pinf = pack_points(Ps)
    lk = [rng.randrange(c.n) for _ in range(n)]
    xy, inf = eng.lincomb(curve, pack_scalars(lk), pxy, pinf)
    out[curve + "_lc_xy"], out[curve + "_lc_inf"] = np.asarray(xy), np.asarray(inf)
eng.close()
np.savez(sys.argv[1], **out)
"""


def _run(tmp_path, tag, inline):
    env = dict(os.environ)
    env.pop("ECG_INLINE_LOOPS", None)
    if not inline:
        env["ECG_INLINE_LOOPS"] = "0"
    dst = str(tmp_path / f"{tag}.npz")
    paths = [ROOT, os.path.join(ROOT, "elliptic-curves_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")]
    subprocess.run([sys.executable, "-s", "-c", SCRIPT, dst] + paths, env=env, check=True, cwd=str(tmp_path), timeout=900)
    return np.load(dst)


def test_call_based_loop_kernels_match_the_inlined_ones(tmp_path):
    import ecref
    from helpers import edge_scalars, pack_scalars
    import pyref
    import random

    inl = _run(tmp_path, "inlined", True)
    call = _run(tmp_path, "calls", False)
    assert sorted(inl.files) == sorted(call.files)
    for k in inl.files:
        assert np.array_equal(inl[k], call[k]), f"ECG_INLINE_LOOPS=0 changes {k}"
    # and both are right: k*G against the C restatement of the reference
    for curve in ("k256", "p256"):
        c = pyref.CURVES[curve]
        rng = random.Random(7)
        ks = edge_scalars(c) + [rng.randrange(c.n) for _ in range(3000)]
        r_xy, r_inf = ecref.mul_gen_batch(curve, pack_scalars(ks), nthreads=8)
        assert np.array_equal(call[curve + "_kg_xy"].reshape(-1), r_xy.reshape(-1))
        assert np.array_equal(call[curve + "_kg_inf"], r_inf)
