"""Sequence-parallel groups on the kernel path across GPUs: ``GPT(sequence_parallel_size=2)`` at world size 4, so
each group of two GPUs holds S_loc = 256 rows of a 512-token context and runs the ``SP`` flash kernels over the
group all-gather and reduce-scatter, against the reference path on the same ranks."""
import pytest
import torch


@pytest.mark.multigpu
@pytest.mark.gpu
def test_multigpu_gpt_groups_kernel_path_matches_reference():
    if torch.cuda.device_count() < 4:
        pytest.skip("needs >= 4 GPUs")
    from mp_util import run_workers
    res = run_workers(4, "sp_group_cases", "kernel_gpt_groups_match_reference", args=(2, 512, 2), cuda=True,
                      timeout=600)
    assert [r["group"] for r in res] == [0, 0, 1, 1], res
    assert res[0]["group_ref"] == res[1]["group_ref"] and res[2]["group_ref"] == res[3]["group_ref"], res
    assert res[0]["group_ref"] != res[2]["group_ref"], res                # two groups, two batches
