"""The fused spline kernel's compiled code (csrc/nfb_fused_rqs.cu, both `fused_rqs_kernel` instances), cross-compiled
for sm_90a: every record's `wgmma` are issued as one straight chain.  ptxas lowers a predicated `wgmma` to a branch
around it, puts it in a basic block of its own, injects a `warpgroup.arrive` in front and gives it its own scoreboard
(`gsb0`), which leaves the tensor core idle between products; these checks keep that from coming back."""
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
    """(ptxas resource lines, SASS instructions) per fused_rqs_kernel instance."""
    out = str(tmp_path_factory.mktemp("fused_sass") / "nfb_fused_rqs.cubin")
    p = subprocess.run([NVCC, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-cubin", "-Xptxas", "-v",
                        "-o", out, "nfb_fused_rqs.cu"], cwd=CSRC, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-4000:]
    resources, fn = {}, None
    for line in p.stderr.splitlines():
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
        ins = []
        for line in part.splitlines():
            m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", line)
            if m:
                ins.append(re.sub(r"\s+", " ", m.group(1)))
        code[name] = ins
    kernels = sorted(n for n in code if "fused_rqs_kernel" in n)
    assert len(kernels) == 2, sorted(code)
    return {k: (resources.get(k), code[k]) for k in kernels}


def hgmma(ins):
    return [i for i, s in enumerate(ins) if "HGMMA" in s]


def test_no_stack_frame_or_spills(compiled):
    for name, (res, _) in compiled.items():
        assert res == (0, 0, 0), f"{name}: stack frame / spill stores / spill loads = {res}"


def chains(ins):
    """The HGMMA indices of each chain: from one commit group's first wgmma to the one that carries its scoreboard (gsb0).
    (The empty commit groups that stand in for skipped records are single HGMMA with no accumulator, .F16 RZ.)"""
    out, cur = [], []
    for i in hgmma(ins):
        cur.append(i)
        if "gsb0" in ins[i]:
            out.append(cur)
            cur = []
    assert not cur, "a wgmma chain without a scoreboard at its end"
    return [c for c in out if ".F32" in ins[c[0]]]


def test_record_chains_have_no_branch(compiled):
    for name, (_, ins) in compiled.items():
        cs = chains(ins)
        assert cs, name
        for c in cs:
            # a record is at least one K = 16 slab of three products (W_hi A_hi, W_hi A_lo, W_lo A_hi)
            assert len(c) >= 3, f"{name}: a chain of {len(c)}: {[ins[i] for i in c]}"
            for a, b in zip(c, c[1:]):
                gap = [s for s in ins[a + 1:b] if re.search(r"\b(BRA|BRX|JMP|JMX|CALL|RET|EXIT|WARPGROUP\.\w+)\b", s)]
                assert not gap, f"{name}: a branch or warpgroup fence inside a wgmma chain between\n  {ins[a]}\n  {ins[b]}\n  {gap}"
                assert ins[a].split()[0] == ins[b].split()[0], f"{name}: one chain, two shapes: {ins[a]} / {ins[b]}"


def test_one_warpgroup_arrive_per_chain(compiled):
    for name, (_, ins) in compiled.items():
        n_mma = len(hgmma(ins))
        n_arrive = sum("WARPGROUP.ARRIVE" in s for s in ins)
        assert 4 * n_arrive <= n_mma, f"{name}: {n_arrive} warpgroup.arrive for {n_mma} HGMMA"


def test_final_layer_is_one_n96_product_per_slab(compiled):
    for name, (_, ins) in compiled.items():
        shapes = {re.match(r"(?:@\S+ )?HGMMA\.(\d+x\d+x\d+)", ins[i]).group(1) for i in hgmma(ins)}
        assert "64x96x16" in shapes, f"{name}: {sorted(shapes)}"
        assert "64x48x16" not in shapes, f"{name}: {sorted(shapes)}"
