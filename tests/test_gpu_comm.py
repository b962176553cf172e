"""sm_90a communication kernels vs NCCL (multi-GPU: skipped on machines with fewer than 2 GPUs)."""
import pytest
import torch

from mp_util import run_workers

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def _world():
    n = torch.cuda.device_count()
    return 8 if n >= 8 else (4 if n >= 4 else 2)


def test_runtime_setup():
    res = run_workers(_world(), "gpu_cases", "runtime_setup", cuda=True, timeout=300)
    print("symmetric runtime:", res[0])
    assert all(r["gran"] >= (1 << 21) for r in res)


def test_allreduce_matches_nccl():
    res = run_workers(_world(), "gpu_cases", "allreduce_matches_nccl",
                      (["oneshot", "twoshot", "nvls"],), cuda=True, timeout=600)
    assert all(r > 0 for r in res)


def test_broadcast():
    assert all(run_workers(_world(), "gpu_cases", "broadcast_matches", cuda=True, timeout=300))


@pytest.mark.parametrize("opt,dtype,algo", [
    ("sgd", "fp32", "oneshot"), ("sgd", "bf16", "twoshot"), ("sgd_nesterov", "fp32", "twoshot"),
    ("adam", "fp32", "oneshot"), ("adamw", "fp32", "nvls"), ("sgd", "bf16", "nvls"),
])
def test_fused_optimizer(opt, dtype, algo):
    res = run_workers(_world(), "gpu_cases", "fused_optimizer_matches_torch", (opt, dtype, algo),
                      cuda=True, timeout=300)
    print("algorithms:", res[0])


def test_lstm_dp_training():
    res = run_workers(_world(), "gpu_cases", "lstm_dp_training", cuda=True, timeout=300)
    print("algorithms:", res[0])


def test_stress_flag_reuse():
    assert all(run_workers(_world(), "gpu_cases", "stress_flag_reuse", (2000,), cuda=True,
                           timeout=600))


def test_watchdog_reports_missing_rank(monkeypatch):
    monkeypatch.setenv("B200DP_KERNEL_TIMEOUT_S", "3")
    res = run_workers(2, "gpu_cases", "watchdog_timeout", cuda=True, timeout=300)
    assert all(res)


def test_native_collectives_match_nccl():
    assert all(run_workers(_world(), "gpu_cases", "native_collectives_match_nccl", cuda=True, timeout=600))


def test_sync_bn_kernel_path():
    assert all(run_workers(_world(), "gpu_cases", "sync_bn_kernel_path", cuda=True, timeout=300))


def test_fused_engine_cuda_graph():
    res = run_workers(_world(), "gpu_cases", "fused_engine_cuda_graph", cuda=True, timeout=600)
    print("losses:", res[0])


def test_model_to_after_wrap():
    res = run_workers(_world(), "gpu_cases", "model_to_after_wrap", cuda=True, timeout=300)
    assert all(r >= 1 for r in res), res      # the engine had to re-home at least one parameter


def test_init_shutdown_cycles():
    assert all(run_workers(_world(), "gpu_cases", "init_shutdown_cycles", cuda=True, timeout=600))


def test_allreduce_large():
    assert all(run_workers(_world(), "gpu_cases", "allreduce_large", cuda=True, timeout=900))


@pytest.mark.parametrize("wire", ["bf16", "fp16"])
def test_compression_runs_on_the_fused_engine(wire):
    assert all(run_workers(_world(), "gpu_cases", "compressed_engine", (wire,), cuda=True, timeout=300))
