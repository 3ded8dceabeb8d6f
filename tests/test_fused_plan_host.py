"""The fused spline kernel's weight-stream planner (csrc/nfb_fused_plan.h), compiled for the host by tests/native: slice
ownership, step table and record halves for MADE masks built by the reference's rules, and for unmasked nets."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT

SO = os.path.join(ROOT, "tests", "native", "_fused_plan_host_check.so")
FIRST, LAST, QUAD, SKIP, HALF = 1, 2, 4, 8, 16
STEP = np.dtype([("bytes16", "<u2"), ("n8", "u1"), ("kc", "u1"), ("flags", "u1"), ("kc1", "u1"), ("flags1", "u1"),
                 ("pad", "u1")])


@pytest.fixture(scope="module")
def planlib():
    src = os.path.join(ROOT, "tests", "native", "fused_plan_host_check.cu")
    hdr = os.path.join(ROOT, "normalizing-flows_b200/csrc/nfb_fused_plan.h")
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-o", SO, src])
    return C.CDLL(SO)


def made_masks(D, H, n_blocks, permute_mask, seed=0):
    """MaskedLinear masks of the reference's MADE (nets/made.py: input degrees 1..D, optionally permuted; hidden degrees
    arange(H) % max(1, D-1) + min(1, D-1) with >= masks; output rows of feature t get degree in_deg[t], strict >)."""
    in_deg = np.arange(1, D + 1)
    if permute_mask:
        in_deg = in_deg[np.random.default_rng(seed).permutation(D)]
    hid = np.arange(H) % max(1, D - 1) + min(1, D - 1)
    m_init = (hid[:, None] >= in_deg[None, :]).astype(np.float32)
    m_hid = (hid[:, None] >= hid[None, :]).astype(np.float32) if n_blocks else None
    out_deg = np.repeat(in_deg, 23)
    m_fin = (out_deg[:, None] > hid[None, :]).astype(np.float32)
    return m_init, m_hid, m_fin


def plan(lib, H, D, n_blocks, masks):
    m_init, m_hid, m_fin = masks if masks is not None else (None, None, None)
    vp = lambda a: None if a is None else np.ascontiguousarray(a, np.float32).ctypes.data_as(C.c_void_p)
    keep = [m_init, m_hid, m_fin]  # noqa: F841  (alive across the call)
    own = np.zeros(4, np.int32)
    nbytes = C.c_longlong(0)
    steps = np.zeros(4096, STEP)
    recs, recs_lo = np.zeros((8192, 5), np.int64), np.zeros(8192, np.int64)
    n_recs = C.c_int(0)
    n = lib.fused_plan_host_check(H, D, D, 1 + 2 * n_blocks, vp(m_init), vp(m_hid), vp(m_fin),
                                  own.ctypes.data_as(C.c_void_p), C.byref(nbytes), len(steps),
                                  steps.ctypes.data_as(C.c_void_p), len(recs), recs.ctypes.data_as(C.c_void_p),
                                  recs_lo.ctypes.data_as(C.c_void_p), C.byref(n_recs))
    assert n > 0
    return own.reshape(2, 2), nbytes.value, steps[:n], recs[:n_recs.value], recs_lo[:n_recs.value]


def needs(H, masks):
    """[ns][ns] non-zero blocks of the hidden-to-hidden GEMMs, hidden units sorted by degree (stable)."""
    ns = H // 64
    if masks is None or masks[1] is None:
        return np.ones((ns, ns), bool)
    m_init, m_hid, _ = masks
    perm = np.argsort(m_init.sum(1), kind="stable")
    m = m_hid[np.ix_(perm, perm)] != 0
    return m.reshape(ns, 64, ns, 64).any(axis=(1, 3))


def walk_hidden(steps, own, ns, n_hidden):
    """Consume the hidden GEMMs' steps as the kernel's two warpgroups do; per GEMM: the (slice, K-chunk) blocks each
    warpgroup multiplies, in order, and the records."""
    gemms, s = [], 0
    for ph in range(n_hidden):
        onto = ph > 0 and ph % 2 == 0
        blocks, done, recs = [[], []], [False, False], []
        q = [0, 0]
        nrun = [max(1, int((own[w] >= 0).sum())) for w in range(2)]
        while not all(done):
            st = steps[s]
            s += 1
            recs.append(st)
            for w in range(2):
                assert not done[w], "the warpgroups leave a GEMM on different records"
                kc, fl = (int(st["kc"]), int(st["flags"])) if w == 0 else (int(st["kc1"]), int(st["flags1"]))
                j = int(own[w][q[w]]) if q[w] < 2 else -1
                if not fl & SKIP:
                    assert j >= 0
                    live = [b for b in blocks[w] if b[0] == j]
                    assert bool(fl & FIRST) == (not live and not onto)
                    blocks[w].append((j, kc))
                if fl & LAST:
                    q[w] += 1
                    done[w] = q[w] == nrun[w]
        gemms.append((blocks, recs))
    return gemms, s


def old_layout(need, ns):
    """Records per hidden GEMM of the parent's packer: slice q paired with q + ceil(ns/2), union of their K-chunks,
    both halves streamed whether zero or not."""
    half = (ns + 1) // 2
    recs, halves = 0, 0
    for q in range(half):
        jb = q + half
        for kc in range(ns):
            if kc == 0 or need[q][kc] or (jb < ns and need[jb][kc]):
                recs += 1
                halves += 2 if jb < ns else 1
    return recs, halves


def fewest_records(need, ns):
    """Records of a hidden GEMM under the best ownership with at most ceil(ns/2) slices per warpgroup."""
    per_slice = [1 + int(need[j][1:].sum()) for j in range(ns)]
    half = (ns + 1) // 2
    best = None
    for m in range(1 << ns):
        wg1 = [j for j in range(ns) if m >> j & 1]
        if len(wg1) > half or ns - len(wg1) > half:
            continue
        r = max(sum(per_slice[j] for j in range(ns) if j not in wg1), sum(per_slice[j] for j in wg1))
        best = r if best is None else min(best, r)
    return best


CASES = [(D, H, pm) for D in (5, 64) for H in (64, 128, 192, 256) for pm in (False, True)]


@pytest.mark.parametrize("D,H,permute_mask", CASES)
@pytest.mark.parametrize("n_blocks", [0, 2])
def test_made_plan_covers_every_block_once(planlib, D, H, permute_mask, n_blocks):
    masks = made_masks(D, H, n_blocks, permute_mask)
    ns, n_hidden = H // 64, 1 + 2 * n_blocks
    own, nbytes, steps, recs, recs_lo = plan(planlib, H, D, n_blocks, masks)
    half = (ns + 1) // 2
    owned = sorted(int(j) for j in own.ravel() if j >= 0)
    assert owned == list(range(ns))
    for w in range(2):
        n = int((own[w] >= 0).sum())
        assert n <= half and (n == 0 or own[w][0] >= 0)
    need = needs(H, masks)
    gemms, s_end = walk_hidden(steps, own, ns, n_hidden)
    off = 0
    rec_iter = iter(zip(recs, recs_lo))
    for ph, (blocks, srecs) in enumerate(gemms):
        kcs = 1 if ph == 0 else ns
        want = sorted((j, kc) for j in range(ns) for kc in range(kcs) if kc == 0 or need[j][kc])
        got = sorted(blocks[0] + blocks[1])
        assert got == want, "every non-zero block exactly once"
        for w in range(2):
            for j in set(b[0] for b in blocks[w]):
                ks = [kc for jj, kc in blocks[w] if jj == j]
                assert ks == sorted(ks) and ks[0] == 0
        for st in srecs:
            live = [w for w in range(2) if not int(st["flags" if w == 0 else "flags1"]) & SKIP]
            single = bool(int(st["flags"]) & HALF)
            assert bool(int(st["flags1"]) & HALF) == single
            assert len(live) == (1 if single else 2), "no streamed half is all zero"
            tot = 64 if single else 128
            assert int(st["bytes16"]) * 16 == tot * 256 and st["n8"] == 8
            # the record's halves, in the order the kernel addresses them (warpgroup 0's first; a single half at 0)
            for i, w in enumerate(live):
                r, lo = next(rec_iter)
                kc = int(st["kc" if w == 0 else "kc1"])
                assert r[0] == ph and r[2] == 64 and r[3] == kc
                assert r[4] == off + i * 64 * 128 and lo == r[4] + tot * 128
                assert r[1] % 64 == 0 and (r[1] // 64) in [int(j) for j in own[w] if j >= 0]
            off += tot * 256
        if ph == 0:
            assert sum(int(st["bytes16"]) * 16 for st in srecs) == H * 256   # the LU fold overwrites exactly this much
        else:
            assert len(srecs) == fewest_records(need, ns), "the ownership minimises the records"
    # final layer: every record carries two chunks, and the stream ends with it
    for st in steps[s_end:]:
        assert not int(st["flags"]) & HALF and st["kc"] == st["kc1"] and st["n8"] == 6
    assert nbytes == off + sum(int(st["bytes16"]) * 16 for st in steps[s_end:])


@pytest.mark.parametrize("D,H", [(D, H) for D in (5, 64) for H in (64, 128, 192, 256)])
def test_dense_plan_is_the_contiguous_split(planlib, D, H):
    ns = H // 64
    half = (ns + 1) // 2
    own, nbytes, steps, _, _ = plan(planlib, H, D, 2, None)
    pad = lambda js: js + [-1] * (2 - len(js))
    assert [list(own[0]), list(own[1])] == [pad(list(range(half))), pad(list(range(half, ns)))]
    # today's record sequence: per GEMM, pair (q, q + half) over every K-chunk; a pair without a second slice streams
    # warpgroup 0's half alone
    expect = []
    for ph in range(5):
        for q in range(half):
            for kc in range(1 if ph == 0 else ns):
                expect.append((128 if q + half < ns else 64, kc))
    got = [(int(st["bytes16"]) // 16, int(st["kc"])) for st in steps[:len(expect)]]
    assert got == expect
    for st in steps[:len(expect)]:
        if int(st["bytes16"]) // 16 == 128:
            assert st["kc1"] == st["kc"] and not (int(st["flags"]) | int(st["flags1"])) & SKIP


def test_flagship_stream_is_balanced(planlib):
    """D = 64, H = 256, 2 residual blocks: the block-triangular hidden masks have 10 non-zero blocks of 16; warpgroups
    owning {0, 3} / {1, 2} multiply 5 each: 5 records per 256 -> 256 GEMM, against 7 for the contiguous pairing."""
    D, H = 64, 256
    masks = made_masks(D, H, 2, False)
    own, nbytes, steps, _, _ = plan(planlib, H, D, 2, masks)
    assert [list(own[0]), list(own[1])] == [[0, 3], [1, 2]]
    need = needs(H, masks)
    assert int(need.sum()) == 10
    gemms, _ = walk_hidden(steps, own, 4, 5)
    assert [len(r) for _, r in gemms] == [2, 5, 5, 5, 5]
    lu = 16 * 1024
    assert (lu + nbytes) // 1024 == 1680
    old_recs, _ = old_layout(need, 4)
    assert old_recs == 7
    final = nbytes - sum(int(st["bytes16"]) * 16 for _, r in gemms for st in r)
    assert (lu + 64 * 1024 + 4 * old_recs * 32 * 1024 + final) // 1024 == 1936
    # final layer: the K = 16 slabs a chunk's features reach form a prefix of its last K-chunk; the rest are skipped
    _, s_end = walk_hidden(steps, own, 4, 5)
    halves = slabs = 0
    for st in steps[s_end:]:
        for fl in (int(st["flags"]), int(st["flags1"])):
            if not fl & SKIP:
                halves += 1
                slabs += 4 - ((fl >> 5) & 3)
    assert (halves, slabs) == (80, 272)


def test_dense_final_layer_issues_every_slab(planlib):
    _, _, steps, _, _ = plan(planlib, 256, 64, 2, None)
    assert all((int(st["flags"]) | int(st["flags1"])) >> 5 == 0 for st in steps)
