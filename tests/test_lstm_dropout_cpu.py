"""Inter-layer LSTM dropout without a GPU: the entry script's ``--lstm-dropout`` flag, the model's ``dropout``
argument and the argument checks of ``ops/lstm_rec.py::lstm_stack``."""
import re

import pytest
import torch

from test_app_script import _run


def test_lstm_cpu_stacked_dropout(tmp_path):
    r = _run(["--device", "cpu", "--lstm-layers", "2", "--lstm-dropout", "0.2", "--epochs", "1",
              "--max-steps", "2"], cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr[-2000:]
    out = r.stdout
    assert len(re.findall(r"epoch: 0, train_loss: [\d.e-]+", out)) == 1
    assert len(re.findall(r"epoch: 0, test_loss: [\d.e-]+", out)) == 1
    assert re.search(r"device: 0, avg_time_per_epoch:[\d.]+", out)
    assert re.search(r"total training time in minutes: [\d.e-]+", out)


def test_model_dropout_keeps_parameters():
    from distributed_torch_horovod_gcp_b200.models import LSTM
    m = LSTM(23, 10, 1, 256, n_layers=2, dropout=0.3)
    ref = LSTM(23, 10, 1, 256, n_layers=2)
    assert m.lstm.dropout == 0.3 and ref.lstm.dropout == 0
    assert {k: v.shape for k, v in m.state_dict().items()} == {k: v.shape for k, v in ref.state_dict().items()}


@pytest.mark.parametrize("p", [-0.1, 1.5])
def test_lstm_stack_rejects_dropout_outside_unit_interval(p):
    from distributed_torch_horovod_gcp_b200.ops import lstm_rec
    x, h = torch.zeros(2, 3, 23), torch.zeros(2, 2, 256)
    weights = [torch.zeros(4 * 256, 23), torch.zeros(4 * 256, 256), torch.zeros(4 * 256), torch.zeros(4 * 256),
               torch.zeros(4 * 256, 256), torch.zeros(4 * 256, 256), torch.zeros(4 * 256), torch.zeros(4 * 256)]
    with pytest.raises(ValueError, match="dropout"):
        lstm_rec.lstm_stack(x, h, h, weights, 2, False, dropout=p)
