"""The fused spline kernel's final layer runs on two roles (csrc/nfb_fused_rqs.cu): warpgroup 0 walks the final layer's
records and multiplies both halves, warpgroup 1 evaluates the splines and moves its ring cursors (slot, parity, step index)
past those records by arithmetic.  This walks the planner's step tables (csrc/nfb_fused_plan.h, compiled for the host)
as the two roles do and checks that they agree: a disagreement would leave warpgroup 1 waiting on the wrong ring slot in
the next hidden GEMM."""
import numpy as np
import pytest

from test_fused_plan_host import FIRST, HALF, LAST, QUAD, SKIP, STEP, made_masks, plan, planlib  # noqa: F401

SLOTS = 3


def step_table(steps, has_lu):
    """The table a unit walks: the LU record in front of the block's (nfb_api.cu lu_step)."""
    if not has_lu:
        return steps
    lu = np.zeros(1, STEP)
    lu["bytes16"], lu["n8"] = 64 * 16, 8
    lu["flags"] = FIRST | LAST | QUAD | HALF
    lu["flags1"] = FIRST | LAST | QUAD | HALF | SKIP
    return np.concatenate([lu, steps])


class Cursor:
    """slot / parity / step index of one consumer warpgroup, moved as run_records moves them."""

    def __init__(self, table, lu_steps):
        self.table, self.lu_steps = table, lu_steps
        self.slot = self.par = self.sidx = self.count = 0

    def new_unit(self):
        self.sidx = 0

    def record(self):
        st = self.table[self.sidx]
        self.sidx = self.lu_steps if self.sidx + 1 == len(self.table) else self.sidx + 1
        self.slot += 1
        if self.slot == SLOTS:
            self.slot, self.par = 0, self.par ^ 1
        self.count += 1
        return st

    def run(self, flag_field):
        """One run of records, until the one marked last in `flag_field`; returns them."""
        out = []
        while True:
            out.append(self.record())
            if int(out[-1][flag_field]) & LAST:
                return out

    def skip_final(self):
        """Warpgroup 1 in the final layer: the records from here to the end of the table."""
        n = len(self.table) - self.sidx
        adv = self.slot + n
        self.slot, self.par, self.sidx = adv % SLOTS, self.par ^ ((adv // SLOTS) & 1), self.lu_steps
        self.count += n
        return n

    def state(self):
        return self.slot, self.par, self.sidx, self.count


def walk_unit(table, own, has_lu, n_hidden, n_pairs, passes, cur):
    """One (layer, tile) unit on both warpgroups; cur = their cursors (carried from unit to unit, as in the kernel)."""
    for c in cur:
        c.new_unit()
    if has_lu:
        for w, c in enumerate(cur):
            c.run("flags1" if w else "flags")
    for _ in range(passes):
        for ph in range(n_hidden):
            for w, c in enumerate(cur):
                for q in range(2):
                    if q == 0 or own[w][q] >= 0:
                        c.run("flags1" if w else "flags")
            assert cur[0].state() == cur[1].state(), "the warpgroups leave a hidden GEMM on different records"
        first_final = cur[0].sidx
        walked = 0
        for _ in range(n_pairs):
            recs = cur[0].run("flags")
            walked += len(recs)
            for st in recs[:-1]:
                assert not int(st["flags1"]) & LAST
            assert int(recs[-1]["flags1"]) & LAST, "a pair ends on one record for both halves"
            for st in recs:
                assert not (int(st["flags"]) | int(st["flags1"])) & HALF and st["n8"] == 6
        assert cur[1].sidx == first_final
        assert cur[1].skip_final() == walked, "warpgroup 1 skips what warpgroup 0 consumed"
        assert cur[0].state() == cur[1].state()
    # the producer streams the LU record once and the block's records once per pass
    return has_lu + passes * (len(table) - has_lu)


def check(planlib, H, n_in, T, n_blocks, masks, passes_of):
    own, _, steps, _, _ = plan(planlib, H, n_in, n_blocks, masks)
    n_pairs = (((T + 1) // 2 + 1) & ~1) // 2   # as nfb_api.cu build_fused: two features per chunk, chunks in pairs
    for has_lu in (0, 1):
        table = step_table(steps, has_lu)
        for passes in passes_of:
            cur = [Cursor(table, has_lu), Cursor(table, has_lu)]
            streamed = 0
            for _ in range(3):   # consecutive units: the slot and parity carry over, the step index starts again
                streamed += walk_unit(table, own, has_lu, 1 + 2 * n_blocks, n_pairs, passes, cur)
                assert cur[0].count == streamed, "the consumers take exactly what the producer streams"


@pytest.mark.parametrize("permute_mask", [False, True])
@pytest.mark.parametrize("n_blocks", [0, 1, 2, 3])
@pytest.mark.parametrize("H", [64, 128, 192, 256])
def test_autoregressive_plans(planlib, H, n_blocks, permute_mask):
    for D in range(1, 65):
        check(planlib, H, D, D, n_blocks, made_masks(D, H, n_blocks, permute_mask, seed=D), (1, D))


@pytest.mark.parametrize("n_blocks", [0, 2])
@pytest.mark.parametrize("H", [64, 128, 192, 256])
def test_unmasked_plans(planlib, H, n_blocks):
    """Coupled blocks: an unmasked conditioner; the plan depends on the transformed feature count alone."""
    for T in range(1, 65):
        check(planlib, H, T, T, n_blocks, None, (1,))
