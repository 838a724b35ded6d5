"""Two properties of the inline-PTX carry-chain code that only the device build can break, checked on the PTX the
library's own flags produce (no GPU needed: nvcc cross-compiles).

 * No register aliasing inside an asm block.  Every primitive of ecg_prim.cuh writes its outputs only after reading all
   of its inputs within one instruction, or reads them again later (mad_acc3: the multiplicands feed two instructions).
   If the compiler puts an input in an output's register — legal unless the output is early-clobber — a later
   instruction of the block reads the overwritten value.  This is the sm2 / P-192 bug mad_acc3x fixes (DESIGN.md §4):
   with -p^-1 mod 2^32 = 1 the Montgomery factor m = c0 shared c0's register.  The scan: within one
   `// begin inline asm` ... `// end inline asm` block, no instruction reads a register an earlier one wrote.
 * Unbroken carry chains.  Every addc / subc / madc must find the carry flag set by a `.cc` instruction earlier in the
   same straight-line stretch: no label, branch, call or return in between."""
import os
import re
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "elliptic-curves_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def _flags():
    import __graft_entry__ as ge

    return [f for f in ge.NVCC_FLAGS if f not in ("-Xcompiler", "-fPIC")]


def _ptx(src, out, defines=(), includes=()):
    cmd = [NVCC] + _flags() + [f"-D{d}" for d in defines] + [f"-I{i}" for i in includes] + ["-ptx", "-o", out, src]
    subprocess.run(cmd, check=True, capture_output=True, timeout=1200)
    with open(out) as f:
        return f.read()


REG = re.compile(r"%[a-z]+\d+")


def _operands(line):
    ins = line.split(";")[0].strip()
    if not ins or ins.startswith("//") or ins.startswith("@"):
        return None, None, []
    parts = ins.split(None, 1)
    if len(parts) < 2:
        return parts[0], None, []
    ops = [o.strip() for o in parts[1].split(",")]
    return parts[0], ops[0], [r for o in ops[1:] for r in REG.findall(o)]


def aliasing_findings(ptx):
    """asm blocks in which an instruction reads a register an earlier instruction of the block wrote"""
    found, block = [], None
    for line in ptx.splitlines():
        s = line.strip()
        if s.startswith("// begin inline asm"):
            block = []
        elif s.startswith("// end inline asm"):
            written = set()
            for op, dst, srcs in block:
                hit = written & set(srcs)
                if hit:
                    found.append("; ".join(f"{o} {d}, {', '.join(r)}" for o, d, r in block))
                    break
                if dst:
                    written.add(dst)
            block = None
        elif block is not None:
            op, dst, srcs = _operands(s)
            if op:
                block.append((op, dst, srcs))
    return found


CARRY_USE = re.compile(r"^(addc|subc|madc)\.")
BARRIER = re.compile(r"^(\$?[A-Za-z_][\w$]*:|bra|call|ret|exit|\}|\{)")


def carry_findings(ptx):
    """carry consumers with no carry producer before them in the same straight-line stretch"""
    found, live, func = [], False, ""
    for line in ptx.splitlines():
        s = line.split("//")[0].strip()
        if not s:
            continue
        if s.startswith(".visible .entry") or s.startswith(".entry") or s.startswith(".func") or s.startswith(".visible .func"):
            func = s
        if BARRIER.match(s) or s.startswith("@"):
            # a guarded instruction may not execute: a carry it would set or use is not part of a straight chain
            if s.startswith("@") and CARRY_USE.match(s.split(None, 1)[1] if " " in s else ""):
                found.append(f"{func}: guarded carry use: {s}")
            live = False if not s.startswith("@") else live
            continue
        op = s.split(None, 1)[0]
        if CARRY_USE.match(op) and not live:
            found.append(f"{func}: {s}")
        if ".cc." in op + ".":
            live = True
    return found


@pytest.fixture(scope="module")
def library_ptx(tmp_path_factory):
    """ecgpu.cu for every curve group and the device test library, compiled to PTX in parallel"""
    d = tmp_path_factory.mktemp("ptx")
    jobs = [(os.path.join(CSRC, "ecgpu.cu"), str(d / f"tu{g}.ptx"), (f"ECG_TU={g}",)) for g in (0, 1, 2, 3, 4)]
    fe_dev = os.path.join(ROOT, "tests", "dev", "fe_dev.cu")
    jobs += [(fe_dev, str(d / "fe_dev_main.ptx"), ()), (fe_dev, str(d / "fe_dev_s1.ptx"), ("DEV_SHAPE=1",))]
    with ThreadPoolExecutor(len(jobs)) as ex:
        res = list(ex.map(lambda j: (os.path.basename(j[1]), _ptx(*j)), jobs))
    return dict(res)


def test_no_register_aliasing_in_asm_blocks(library_ptx):
    for name, ptx in library_ptx.items():
        assert ptx.count("// begin inline asm") > 1000, name  # the primitives are really there
        found = aliasing_findings(ptx)
        assert not found, f"{name}: {len(found)} asm blocks read a register they wrote, e.g. {found[0]}"


def test_carry_chains_are_straight_line(library_ptx):
    for name, ptx in library_ptx.items():
        found = carry_findings(ptx)
        assert not found, f"{name}: {len(found)} carry uses without a producer, e.g. {found[:3]}"


SMALL_TU = r"""
#include "ecg_curves.cuh"
using namespace ecg;
// sm2 and P-192: -p^-1 mod 2^32 = 1, so the Montgomery factor equals the accumulator's low word
__global__ void mont_kernel(const FeN<8>* a, FeN<8>* r, const FeN<6>* b, FeN<6>* s) {
  FeN<8> x = a[threadIdx.x], y = a[threadIdx.x + 1];
  CurveSm2::F::mul(r[threadIdx.x], x, y);
  FeN<6> u = b[threadIdx.x], v = b[threadIdx.x + 1];
  CurveP192::F::mul(s[threadIdx.x], u, v);
}
"""


def test_scan_finds_the_early_clobber_bug(tmp_path):
    """The same scan on a copy of the sources with mad_acc3x (early-clobber outputs) replaced by mad_acc3: the historical
    sm2 / P-192 miscompilation must show up; the unmodified sources are the control"""
    src = tmp_path / "small.cu"
    src.write_text(SMALL_TU)
    assert not aliasing_findings(_ptx(str(src), str(tmp_path / "good.ptx"), includes=(CSRC,)))
    bad = tmp_path / "csrc"
    shutil.copytree(CSRC, bad)
    mont = bad / "ecg_fe_mont.cuh"
    text = mont.read_text()
    assert text.count("mad_acc3x(") >= 5
    mont.write_text(text.replace("mad_acc3x(", "mad_acc3("))
    found = aliasing_findings(_ptx(str(src), str(tmp_path / "bad.ptx"), includes=(str(bad),)))
    assert found, "the scan no longer sees the aliasing mad_acc3 produces for sm2 / P-192"
    assert any(re.match(r"mad\.lo\.cc\.u32 (%r\d+), \1, ", f) for f in found)


def test_carry_scan_sees_a_broken_chain():
    ptx = "\n".join([".visible .entry k(", "{", "add.cc.u32 %r1, %r2, %r3;", "addc.cc.u32 %r4, %r5, %r6;", "$L__BB0_1:",
                     "addc.u32 %r7, %r8, %r9;", "}"])
    assert carry_findings(ptx) == [".visible .entry k(: addc.u32 %r7, %r8, %r9;"]
