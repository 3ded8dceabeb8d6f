"""The fused spline kernel's hidden GEMMs keep their products in flight across record and slice boundaries
(csrc/nfb_fused_rqs.cu, both `fused_rqs_kernel` instances, cross-compiled for sm_90a).

Each consumer warpgroup walks the records of both its output slices of a GEMM as one run: slice 1's first record is
issued while slice 0's last one multiplies, its `wgmma.wait_group 1` completes slice 0, and slice 0's epilogue arithmetic
runs under slice 1's products.  The tensor core drains once per GEMM, before the barrier after which the output is
stored to the A operand with `stmatrix`.  What in the compiled code shows that the schedule survived:

* No `HGMMA.64x8x16 ... RZ` (an empty commit group) follows an m64n64k16 chain before that chain's wait.  A
  `wgmma.commit_group` placed after the join of a record's "products or none" branch closes the chain's group at the end
  of its block and adds a second, empty one; `wait_group 1` then waits for the record's own products.
* A `WARPGROUP.DEPBAR.LE gsb0, 0x1` right after an m64n64k16 chain is followed by the next m64n64k16 chain: records
  overlap.
* Every `WARPGROUP.DEPBAR.LE gsb0, 0x0` after an m64n64k16 chain is followed by a barrier before any further `wgmma`:
  the drain ends a GEMM (or the LU stage), never the first of a warpgroup's two slices.
* The hidden epilogue stores with `STSM`, and ptxas reports no serialised `wgmma`, stack frame or spill.
"""
import os
import re
import shutil
import subprocess

import pytest

from conftest import ROOT

CSRC = os.path.join(ROOT, "normalizing-flows_b200", "csrc")
NVCC = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
CUOBJDUMP = shutil.which("cuobjdump") or (os.path.join(os.path.dirname(NVCC), "cuobjdump") if NVCC else None)

pytestmark = pytest.mark.skipif(not NVCC or not CUOBJDUMP or not os.path.exists(CUOBJDUMP),
                                reason="needs nvcc and cuobjdump")


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    """(ptxas messages, SASS instructions) per fused_rqs_kernel instance."""
    out = str(tmp_path_factory.mktemp("fused_hidden") / "nfb_fused_rqs.cubin")
    p = subprocess.run([NVCC, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-cubin", "-Xptxas", "-v",
                        "-o", out, "nfb_fused_rqs.cu"], cwd=CSRC, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-4000:]
    msgs, fn = {}, None
    for line in p.stderr.splitlines():
        m = re.search(r"(?:function|entry function|properties for) '?(\w+)'?", line)
        if m:
            fn = m.group(1)
        if fn:
            msgs.setdefault(fn, []).append(line)
    sass = subprocess.run([CUOBJDUMP, "-sass", out], capture_output=True, text=True, check=True).stdout
    code = {}
    for part in re.split(r"\n\s*Function : ", sass)[1:]:
        name = part.split("\n", 1)[0].strip()
        code[name] = [re.sub(r"\s+", " ", m.group(1)) for m in
                      (re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", line) for line in part.splitlines()) if m]
    kernels = sorted(n for n in code if "fused_rqs_kernel" in n)
    assert len(kernels) == 2, sorted(code)
    return {k: (msgs.get(k, []), code[k]) for k in kernels}


def is_mma(s):
    return "HGMMA" in s


def is_empty(s):
    return bool(re.search(r"HGMMA\.64x8x16\S* RZ", s))


def is_n64_chain_end(s):
    return "HGMMA.64x64x16.F32" in s and "gsb0" in s


def depbar_count(s):
    m = re.search(r"WARPGROUP\.DEPBAR\.LE gsb0, (0x[0-9a-f]+)", s)
    return int(m.group(1), 16) if m else None


def is_barrier(s):
    return bool(re.search(r"\bBAR\.(SYNC|RED)\b", s))


def prev_index(ins, i, pred):
    return next((j for j in range(i - 1, -1, -1) if pred(ins[j])), None)


def next_index(ins, i, pred):
    return next((j for j in range(i + 1, len(ins)) if pred(ins[j])), None)


def test_no_serialised_wgmma_frame_or_spill(compiled):
    for name, (msgs, _) in compiled.items():
        bad = [m for m in msgs if re.search(r"C7515|C751[0-8]\b|serializ|Performance Loss", m)]
        assert not bad, f"{name}: ptxas serialises wgmma:\n" + "\n".join(bad[:5])
        res = [re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", m) for m in msgs]
        res = [tuple(int(x) for x in m.groups()) for m in res if m]
        assert res and all(r == (0, 0, 0) for r in res), f"{name}: stack frame / spill stores / spill loads = {res}"


def test_no_empty_commit_group_after_a_hidden_chain(compiled):
    for name, (_, ins) in compiled.items():
        bad = []
        for i, s in enumerate(ins):
            if not is_empty(s):
                continue
            j = prev_index(ins, i, lambda t: is_mma(t) or "WARPGROUP.DEPBAR" in t)
            if j is not None and is_n64_chain_end(ins[j]):
                bad.append((ins[j], s))
        assert not bad, f"{name}: {len(bad)} empty commit groups right after an m64n64k16 chain: {bad[:2]}"


def test_hidden_records_overlap(compiled):
    for name, (_, ins) in compiled.items():
        overlapped = 0
        for i, s in enumerate(ins):
            if depbar_count(s) != 1:
                continue
            j, k = prev_index(ins, i, is_mma), next_index(ins, i, is_mma)
            if j is not None and k is not None and is_n64_chain_end(ins[j]) and "HGMMA.64x64x16.F32" in ins[k]:
                overlapped += 1
        assert overlapped >= 1, f"{name}: no wait_group 1 between two m64n64k16 chains"


def test_hidden_gemm_drains_once(compiled):
    for name, (_, ins) in compiled.items():
        drains = 0
        for i, s in enumerate(ins):
            if depbar_count(s) != 0:
                continue
            j = prev_index(ins, i, lambda t: is_mma(t) and not is_empty(t))
            if j is None or "HGMMA.64x64x16" not in ins[j]:
                continue
            drains += 1
            k = next_index(ins, i, lambda t: is_mma(t) or is_barrier(t))
            assert k is None or is_barrier(ins[k]), \
                f"{name}: a wait_group 0 after an m64n64k16 chain is followed by more products ({ins[k]})"
        assert drains >= 1, f"{name}: no wait_group 0 ends a hidden GEMM"


def test_hidden_epilogue_stores_with_stmatrix(compiled):
    for name, (_, ins) in compiled.items():
        stsm = [s for s in ins if s.split()[0].startswith("STSM") or " STSM" in s]
        assert len(stsm) >= 8 and len(stsm) % 8 == 0, f"{name}: {len(stsm)} STSM"
        assert all(".M88.4" in s for s in stsm), f"{name}: {stsm[:4]}"
