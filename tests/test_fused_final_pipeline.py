"""The fused spline kernel's final layer keeps its products in flight across record and pair boundaries
(csrc/nfb_fused_rqs.cu, both `fused_rqs_kernel` instances, cross-compiled for sm_90a).

The product warpgroup alternates two accumulators over the pairs of chunks: it issues the first record of pair c + 1,
waits with `wgmma.wait_group 1` (which completes pair c and leaves that record in flight) and stores pair c to the
staging tiles before it goes on.  What in the compiled code shows that the schedule survived:

* ptxas reports no serialised `wgmma` (C7515 and its kin).  It serialises every `wgmma` of the kernel when something
  other than a `wgmma` defines an accumulator register while products are in flight, which a zero-initialised second
  accumulator, or a register copy between the two, would do.
* Each accumulator's staging stores (the `STS` run that ends in the `BAR.ARV` of the "full" hand-off) follow a
  `WARPGROUP.DEPBAR.LE gsb0, 0x1` whose last `HGMMA` before it is an m64n96k16 chain's: that wait leaves the chain
  outstanding, so the stores run while the next pair's first record multiplies.
* No `HGMMA.64x8x16` right after an m64n96k16 chain.  ptxas closes a commit group at the end of the basic block
  of its last `wgmma`; a `wgmma.commit_group` placed after the join of the slab-count `switch` then becomes a second,
  empty group (an m64n8k16 on RZ), and `wait_group 1` waits for the record's own products instead of the one before.
  So every record commits inside its own case.
* A `DEPBAR` with a count of 0 comes before two stagings at most, one per accumulator after the last pair: the tensor
  core is drained once per pass, not at every pair.
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
    out = str(tmp_path_factory.mktemp("fused_pipeline") / "nfb_fused_rqs.cubin")
    p = subprocess.run([NVCC, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-cubin", "-Xptxas", "-v",
                        "-o", out, "nfb_fused_rqs.cu"], cwd=CSRC, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-4000:]
    msgs = {}
    for line in p.stderr.splitlines():
        m = re.search(r"function '(\S+)'", line)
        if m:
            msgs.setdefault(m.group(1), []).append(line)
    sass = subprocess.run([CUOBJDUMP, "-sass", out], capture_output=True, text=True, check=True).stdout
    code = {}
    for part in re.split(r"\n\s*Function : ", sass)[1:]:
        name = part.split("\n", 1)[0].strip()
        code[name] = [re.sub(r"\s+", " ", m.group(1)) for m in
                      (re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", line) for line in part.splitlines()) if m]
    kernels = sorted(n for n in code if "fused_rqs_kernel" in n)
    assert len(kernels) == 2, sorted(code)
    return {k: (msgs.get(k, []), code[k]) for k in kernels}


def test_no_serialised_wgmma(compiled):
    for name, (msgs, _) in compiled.items():
        bad = [m for m in msgs if re.search(r"C7515|C751[0-8]\b|serializ|Performance Loss", m)]
        assert not bad, f"{name}: ptxas serialises wgmma:\n" + "\n".join(bad[:5])


def depbar_count(s):
    m = re.search(r"WARPGROUP\.DEPBAR\.LE gsb0, (0x[0-9a-f]+)", s)
    return int(m.group(1), 16) if m else None


def staging_blocks(ins):
    """Index of each BAR.ARV whose block (back to the previous barrier) holds at least 24 STS: the product warpgroup's
    "full" arrival after an accumulator went to the staging tiles (12 float2 per half and thread)."""
    out = []
    for i, s in enumerate(ins):
        if not re.search(r"\bBAR\.ARV\b", s):
            continue
        j, sts = i - 1, 0
        while j >= 0 and not re.search(r"\bBAR\.(SYNC|ARV|RED)\b", ins[j]):
            sts += ins[j].split()[0].startswith("STS") or " STS" in ins[j]
            j -= 1
        if sts >= 24:
            out.append(i)
    return out


def before(ins, i, pred):
    return next((ins[j] for j in range(i, -1, -1) if pred(ins[j])), "")


def test_pairs_are_staged_under_the_next_pairs_products(compiled):
    for name, (_, ins) in compiled.items():
        blocks = staging_blocks(ins)
        assert blocks, f"{name}: no staging of a final-layer accumulator found"
        waits = [depbar_count(before(ins, b, lambda s: "WARPGROUP.DEPBAR" in s)) for b in blocks]
        mmas = [before(ins, b, lambda s: "HGMMA" in s) for b in blocks]
        # every staging follows the products of an m64n96k16 chain, never an empty commit group
        assert all("HGMMA.64x96x16" in m for m in mmas), f"{name}: {mmas}"
        # one pair boundary per accumulator with a product group in flight; a full drain only after the last pair
        assert waits.count(1) >= 2, \
            f"{name}: {waits.count(1)} of {len(blocks)} stagings run with a product group in flight"
        assert waits.count(0) <= 2, f"{name}: {waits.count(0)} stagings after a wait_group 0: {waits}"
        assert set(waits) <= {0, 1}, f"{name}: {waits}"


def test_no_empty_commit_group_after_a_final_layer_chain(compiled):
    for name, (_, ins) in compiled.items():
        empty = [i for i, s in enumerate(ins) if re.search(r"HGMMA\.64x8x16\S* RZ", s)]
        after96 = [i for i in empty if "HGMMA.64x96x16" in before(ins, i - 1, lambda s: "HGMMA" in s)]
        assert not after96, f"{name}: {len(after96)} empty commit groups right after an m64n96k16 chain"
