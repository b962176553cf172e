"""Algorithm table (autotuner replacement): pure-function behaviour + derivation from a real sweep."""
import json
import os

from distributed_torch_horovod_gcp_b200.runtime import tuning

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_default_table():
    tuning.reset()
    assert tuning.choose(8, 1024, True) == tuning.ONESHOT
    assert tuning.choose(8, 8 << 10, True) == tuning.ONESHOT
    assert tuning.choose(8, 64 << 10, True) == tuning.NVLS
    assert tuning.choose(8, 64 << 10, False) == tuning.TWOSHOT       # no multicast -> P2P two-shot
    assert tuning.choose(2, 1 << 20, True) == tuning.TWOSHOT
    assert tuning.choose(4, 16 << 20, True) == tuning.NVLS


def test_user_table(tmp_path, monkeypatch):
    f = tmp_path / "t.json"
    f.write_text(json.dumps({"8": {"oneshot_max_bytes": 1 << 20, "prefer": "twoshot"}}))
    monkeypatch.setenv("B200DP_TUNING_FILE", str(f))
    tuning.reset()
    assert tuning.choose(8, 512 << 10, True) == tuning.ONESHOT
    assert tuning.choose(8, 2 << 20, True) == tuning.TWOSHOT
    assert tuning.choose(4, 2 << 20, True) == tuning.NVLS               # other worlds keep defaults
    monkeypatch.delenv("B200DP_TUNING_FILE")
    tuning.reset()


def test_derive_from_measured_sweep():
    # benchmarks/allreduce_sweep.py output recorded on an 8-GPU NVSwitch node with multicast (8x B200)
    rows = json.load(open(os.path.join(ROOT, "tests", "golden", "allreduce_sweep_8gpu.json")))["rows"]
    row = tuning.derive_from_sweep(rows, 8, True)
    assert row["prefer"] == "nvls"                      # NVLS has the highest bus bandwidth at 1 GiB
    assert row["oneshot_max_bytes"] <= 64 << 10         # one-shot never wins above the latency regime
