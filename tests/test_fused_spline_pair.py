"""The fused spline kernel's spline warpgroup takes a final-layer pair of chunks in one go (csrc/nfb_fused_rqs.cu, both
`fused_rqs_kernel` instances, cross-compiled for sm_90a).

Per pair it waits for "full", reads both splines' parameters from the two staging tiles (6 `LDS.128` per tile and
thread), hands the tiles back ("free") and only then evaluates the two splines, as one two-lane `rqs_core_lanes` call
(csrc/nfb_spline.cuh) whose dependent chains ptxas can interleave.  What in the compiled code shows that:

* ptxas reports no spill, no stack frame and no serialised `wgmma`: the two chains fit the consumers' registers.
* In the pair loop (from the `BAR.SYNC` of "full" to the branch back to it) every `LDS.128` comes before the `BAR.ARV` of
  "free", and no `MUFU` does: the product warpgroup may stage the next pair while both splines run.
* One basic block of the loop holds the `MUFU.EX2` of both splines (2 x (2 K softmax terms + 2 softplus), K = 8): the
  two evaluations were not split apart into separate blocks or loop iterations.
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

K = 8
EX2_PER_SPLINE = 2 * K + 2


def barrier_ids():
    """(full, free): the named-barrier IDs of the final layer's hand-off, as the kernel source defines them."""
    src = open(os.path.join(CSRC, "nfb_fused_rqs.cu")).read()
    m = re.search(r"constexpr int kBarStgFull = (\d+), kBarStgFree = (\d+);", src)
    assert m, "kBarStgFull / kBarStgFree not found"
    return int(m.group(1)), int(m.group(2))


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    """(ptxas messages, resources, SASS as (address, instruction)) per fused_rqs_kernel instance."""
    out = str(tmp_path_factory.mktemp("fused_spline_pair") / "nfb_fused_rqs.cubin")
    p = subprocess.run([NVCC, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-cubin", "-Xptxas", "-v",
                        "-o", out, "nfb_fused_rqs.cu"], cwd=CSRC, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-4000:]
    msgs, resources, fn = {}, {}, None
    for line in p.stderr.splitlines():
        m = re.search(r"function '(\S+)'", line)
        if m:
            msgs.setdefault(m.group(1), []).append(line)
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            fn = m.group(1)
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and fn:
            resources[fn] = tuple(int(x) for x in m.groups())
    sass = subprocess.run([CUOBJDUMP, "-sass", out], capture_output=True, text=True, check=True).stdout
    code = {}
    for part in re.split(r"\n\s*Function : ", sass)[1:]:
        name = part.split("\n", 1)[0].strip()
        code[name] = [(int(m.group(1), 16), re.sub(r"\s+", " ", m.group(2))) for m in
                      (re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;", line) for line in part.splitlines()) if m]
    kernels = sorted(n for n in code if "fused_rqs_kernel" in n)
    assert len(kernels) == 2, sorted(code)
    return {k: (msgs.get(k, []), resources.get(k), code[k]) for k in kernels}


def pair_loop(ins):
    """The spline warpgroup's pair loop: from the BAR.SYNC of "full" to the branch back to it (inclusive)."""
    full, _ = barrier_ids()
    syncs = [i for i, (_, s) in enumerate(ins) if re.search(rf"\bBAR\.SYNC\S* {full:#x},", s)]
    assert len(syncs) == 1, f"{len(syncs)} waits for the 'full' barrier"
    head = ins[syncs[0]][0]
    for j in range(syncs[0], len(ins)):
        m = re.search(r"\bBRA\b.*?0x([0-9a-f]+)\b", ins[j][1])
        if m and int(m.group(1), 16) <= head:
            return ins[syncs[0]:j + 1]
    raise AssertionError("no branch back to the 'full' wait")


def basic_blocks(body):
    targets = {int(m.group(1), 16) for _, s in body for m in [re.search(r"\bBRA\b.*?0x([0-9a-f]+)\b", s)] if m}
    blocks, cur = [], []
    for a, s in body:
        if a in targets and cur:
            blocks.append(cur)
            cur = []
        cur.append(s)
        if re.search(r"\b(BRA|BRX|JMP|JMX|CALL|RET|EXIT|BSSY|BSYNC)\b", s):
            blocks.append(cur)
            cur = []
    return blocks + [cur] if cur else blocks


def test_no_spill_and_no_serialised_wgmma(compiled):
    for name, (msgs, res, _) in compiled.items():
        assert res == (0, 0, 0), f"{name}: stack frame / spill stores / spill loads = {res}"
        bad = [m for m in msgs if re.search(r"C7515|C751[0-8]\b|serializ|Performance Loss", m)]
        assert not bad, f"{name}: ptxas serialises wgmma:\n" + "\n".join(bad[:5])


def test_tiles_are_handed_back_before_the_splines(compiled):
    _, free = barrier_ids()
    for name, (_, _, ins) in compiled.items():
        body = [s for _, s in pair_loop(ins)]
        arv = [i for i, s in enumerate(body) if re.search(rf"\bBAR\.ARV {free:#x},", s)]
        assert len(arv) == 1, f"{name}: {len(arv)} 'free' arrivals in the pair loop"
        lds = [i for i, s in enumerate(body) if "LDS.128" in s]
        mufu = [i for i, s in enumerate(body) if "MUFU." in s]
        assert len(lds) == 12, f"{name}: {len(lds)} LDS.128 in the pair loop (both tiles: 2 x 6)"
        assert max(lds) < arv[0], f"{name}: a parameter read after the 'free' arrival"
        assert mufu and min(mufu) > arv[0], f"{name}: spline work before the 'free' arrival"


def test_both_splines_in_one_basic_block(compiled):
    for name, (_, _, ins) in compiled.items():
        ex2 = [sum("MUFU.EX2" in s for s in b) for b in basic_blocks(pair_loop(ins))]
        assert max(ex2) >= 2 * EX2_PER_SPLINE, f"{name}: MUFU.EX2 per basic block of the pair loop: {ex2}"
