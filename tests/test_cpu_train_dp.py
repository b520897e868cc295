"""CPU tests (no GPU) of data-parallel training's host side: who runs which micro-batch of each optimizer step, and
the gradient-exchange kernels' machine code in the built library."""
import re

import pytest

from beat_this_b200 import train as T
from support import sass


@pytest.mark.parametrize("batches, accumulate, world", [
    (5, 2, 2), (5, 3, 2), (8, 8, 8), (10, 4, 3), (7, 3, 1), (9, 8, 4), (1, 1, 1), (17, 8, 5), (16, 8, 8)])
def test_every_micro_batch_is_owned_once_in_dense_slots(batches, accumulate, world):
    groups = T.micro_batch_owners(batches, accumulate, world)
    plan = T.step_plan(batches, accumulate)
    # the groups are step_plan's: consecutive micro-batches up to each step point
    assert len(groups) == len(plan) and sum(len(g) for g in groups) == batches
    assert [sum(len(g) for g in groups[: k + 1]) - 1 for k in range(len(groups))] == plan
    slots = -(-accumulate // world)
    for group in groups:
        assert 1 <= len(group) <= accumulate
        assert len(set(group)) == len(group)  # each (rank, slot) once
        for j, (rank, slot) in enumerate(group):
            assert (rank, slot) == (j % world, j // world) and slot < slots
        for rank in range(world):  # a rank's slots are 0, 1, ... without gaps
            mine = [slot for r, slot in group if r == rank]
            assert mine == list(range(len(mine)))


def test_short_groups_leave_the_last_ranks_idle():
    groups = T.micro_batch_owners(5, 2, 2)
    assert groups == [[(0, 0), (1, 0)], [(0, 0), (1, 0)], [(0, 0)]]  # rank 1 sits out the last step
    groups = T.micro_batch_owners(5, 3, 2)
    assert groups == [[(0, 0), (1, 0), (0, 1)], [(0, 0), (1, 0)]]  # rank 0 runs two micro-batches of the first step
    groups = T.micro_batch_owners(11, 8, 4)
    assert [r for r, _ in groups[1]] == [0, 1, 2]  # rank 3 idles in the 3-batch remainder


@pytest.mark.parametrize("accumulate, world", [(2, 3), (1, 2), (8, 9), (3, 0)])
def test_more_ranks_than_micro_batches_per_step_are_refused(accumulate, world):
    with pytest.raises(ValueError):
        T.micro_batch_owners(10, accumulate, world)
    with pytest.raises(ValueError):
        T.micro_batch_owners(0, accumulate, world)


def test_exchange_kernels_have_no_local_memory_and_add_without_fma(lib_built):
    found, local, ops = set(), [], {}
    fn = None
    for line in sass(lib_built).splitlines():
        if "Function :" in line:
            fn = line.split("Function :")[1].strip()
            fn = next((k for k in ("grad_pack_kernel", "grad_ordered_sum_kernel") if k in fn), None)
            if fn:
                found.add(fn)
        elif fn:
            if re.search(r"\b(STL|LDL)(\.\w+)*\b", line):
                local.append((fn, line.strip()))
            for op in ("FADD", "FFMA", "FMUL"):
                if re.search(rf"\b{op}\b", line):
                    ops.setdefault(fn, set()).add(op)
    assert found == {"grad_pack_kernel", "grad_ordered_sum_kernel"}, found
    assert not local, local
    assert ops.get("grad_ordered_sum_kernel") == {"FADD"}  # fp32 adds only: nothing fused or scaled
    assert "grad_pack_kernel" not in ops  # a copy
