"""Distributed training entry point — same path, same zero-argument invocation and the same
printed lines as the reference script (reference app/torch_train.py:208-312):

    python3 app/torch_train.py                                             (1 GPU)
    bin/horovodrun -np 4 -H localhost:4 python3 app/torch_train.py         (4 GPUs)

With no arguments it trains the reference workload: LSTM(23 -> 256) regressor on the
ES-futures window data, fp32, Adam lr=1e-6, per-rank batch 32, ceil(100 / world) epochs,
gradient averaging through ``hvd.DistributedOptimizer`` and an initial
``hvd.broadcast_parameters`` — but on the H100-native runtime instead of Horovod.

Optional flags / environment variables (all default to the reference behaviour) select the
[DRIVER] benchmark variants from BASELINE.json (``--model resnet18|resnet50|resnet152|
vit_b_16``, ``--dtype bf16``, ``--device cpu`` for the CPU/Gloo plumbing config, …).
"""
import argparse
import datetime
import itertools  # noqa: F401  (kept: part of the reference module namespace)
import math
import os
import sys
import warnings  # noqa: F401

import numpy as np
import torch
from torch import nn
from torch.utils.data import DataLoader

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import distributed_torch_horovod_gcp_b200.torch as hvd  # noqa: E402
from distributed_torch_horovod_gcp_b200.data import (  # noqa: E402,F401
    x_cols, y_cols, read_file_from_aws, reshape_and_scale_data_for_training, TimeSeriesDataSet,
    MinMaxScaler, StandardScaler, ensure_dataset, DeviceBatchLoader, SyntheticImageBatches)
from distributed_torch_horovod_gcp_b200.models import LSTM, build as build_model  # noqa: E402
from distributed_torch_horovod_gcp_b200.utils import getGPUs  # noqa: E402


def parse_args(argv=None):
    env = os.environ.get
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawTextHelpFormatter)
    p.add_argument("--model", default=env("B200DP_MODEL", "lstm"))
    p.add_argument("--epochs", type=int, default=int(env("B200DP_EPOCHS", "100")),
                   help="total epoch budget; divided by the world size like the reference")
    p.add_argument("--batch-size", type=int, default=int(env("B200DP_BATCH", "32")))
    p.add_argument("--lr", type=float, default=float(env("B200DP_LR", "1e-6")))
    p.add_argument("--window", type=int, default=10)
    p.add_argument("--device", default=env("B200DP_DEVICE", "auto"), choices=["auto", "cuda", "cpu"])
    p.add_argument("--dtype", default=env("B200DP_DTYPE", "fp32"), choices=["fp32", "bf16"])
    p.add_argument("--max-steps", type=int, default=int(env("B200DP_MAX_STEPS", "0")),
                   help="stop each epoch after this many steps (0 = full epoch)")
    p.add_argument("--loader", default=env("B200DP_LOADER", "auto"),
                   choices=["auto", "device", "dataloader"],
                   help="'dataloader' = the reference's DataLoader+DistributedSampler path")
    p.add_argument("--image-size", type=int, default=int(env("B200DP_IMAGE_SIZE", "0")))
    p.add_argument("--num-classes", type=int, default=int(env("B200DP_NUM_CLASSES", "0")))
    p.add_argument("--steps-per-epoch", type=int, default=int(env("B200DP_STEPS_PER_EPOCH", "20")),
                   help="synthetic image models only")
    p.add_argument("--no-validate", action="store_true")
    p.add_argument("--cuda-graph", action="store_true",
                   default=env("B200DP_CUDA_GRAPH", "0") == "1",
                   help="capture the whole training step (fwd+bwd+fused allreduce/update) in one "
                        "CUDA graph; H100-first answer for the launch-bound LSTM config")
    p.add_argument("--data", default=env("B200DP_DATA", "data_es.csv"))
    return p.parse_args(argv)


if __name__ == "__main__":
    args = parse_args()
    # intialize the runtime (Horovod: hvd.init())
    hvd.init()

    # to handle dynamically updating GPUs: enumerate before any CUDA context exists
    os.environ.setdefault("CUDA_DEVICE_ORDER", "PCI_BUS_ID")
    gpus = getGPUs()
    device_number = hvd.rank()

    use_cuda = torch.cuda.is_available() and args.device != "cpu"
    if not use_cuda and args.device != "cpu" and os.environ.get("B200DP_ALLOW_CPU", "0") != "1":
        print("Needs a GPU to run!")
        exit()

    epochs = args.epochs
    # adjust number of epochs based on number of GPUs.
    epochs = int(math.ceil(epochs / hvd.size()))
    window_length = args.window

    # Pin GPU to be used to process local rank (one GPU per process)
    if use_cuda:
        torch.cuda.set_device(hvd.local_rank())
        _DEVICE = torch.device("cuda:{}".format(str(torch.cuda.current_device())))
    else:
        _DEVICE = torch.device("cpu")

    if device_number == 0:
        print("horovod has distributed to the following devices: {}"
              .format(["{}, device_id: cuda:{}".format(gpu.name, gpu.id) for gpu in gpus]),
              flush=True)

    print(f"this process is using device - {_DEVICE}", flush=True)

    is_lstm = args.model.lower() == "lstm"
    compute_dtype = torch.bfloat16 if args.dtype == "bf16" else torch.float32

    if is_lstm:
        df, source = ensure_dataset(args.data, rank=hvd.rank(),
                                    decide=(lambda v: hvd.broadcast_object(v, 0)) if hvd.size() > 1 else None)
        if hvd.size() > 1:
            hvd.barrier()
        x_train, x_test, y_train, y_test, scaler = reshape_and_scale_data_for_training(
            df, window_length, x_cols, y_cols, y_len=1, scale=True, backend='torch')

        loader_kind = args.loader
        if loader_kind == "auto":
            loader_kind = "device" if use_cuda else "dataloader"
        if loader_kind == "device":
            # H100-first: the whole (small) dataset is device resident; same sharded permutation
            # as DistributedSampler(seed=0) and, like the reference, set_epoch is never called.
            train_loader = DeviceBatchLoader(x_train, y_train, args.batch_size,
                                             num_replicas=hvd.size(), rank=hvd.rank(),
                                             device=_DEVICE)
            test_loader = [(x_test.to(_DEVICE), y_test.to(_DEVICE))]
        else:
            train_sampler = torch.utils.data.distributed.DistributedSampler(
                TimeSeriesDataSet(x_train, y_train), num_replicas=hvd.size(), rank=hvd.rank())
            nw = 4 if use_cuda else 0
            train_loader = DataLoader(TimeSeriesDataSet(x_train, y_train),
                                      batch_size=args.batch_size, pin_memory=use_cuda,
                                      num_workers=nw, sampler=train_sampler)
            test_loader = DataLoader(TimeSeriesDataSet(x_test, y_test), batch_size=len(x_test),
                                     shuffle=True, pin_memory=use_cuda, num_workers=nw)

        model = LSTM(n_features=23, window_size=window_length, output_size=1, h_size=256,
                     device=_DEVICE)
        optimizer = torch.optim.Adam(model.parameters(), lr=args.lr)
        loss_fn = nn.MSELoss(reduction="mean")
    else:
        small = args.model.lower().replace("-", "").replace("_", "") == "resnet18" and not use_cuda
        image_size = args.image_size or (32 if small else 224)
        num_classes = args.num_classes or (10 if small else 1000)
        kw = {"num_classes": num_classes}
        if "resnet" in args.model.lower():
            kw["small_input"] = image_size <= 64
        else:
            kw["image_size"] = image_size
        model = build_model(args.model, **kw).to(_DEVICE)
        if compute_dtype != torch.float32:
            model = model.to(compute_dtype)
        if use_cuda:
            model = model.to(memory_format=torch.channels_last)
        batches = SyntheticImageBatches(args.batch_size, (3, image_size, image_size), num_classes,
                                        _DEVICE, compute_dtype, channels_last=use_cuda,
                                        seed=hvd.rank())

        class _SynthLoader:
            def __iter__(self_inner):
                for _ in range(args.steps_per_epoch):
                    yield batches.next()
        train_loader = _SynthLoader()
        test_loader = [batches.next()]
        lr = args.lr if args.lr != 1e-6 else 0.1
        optimizer = torch.optim.SGD(model.parameters(), lr=lr, momentum=0.9, weight_decay=1e-4)
        loss_fn = nn.CrossEntropyLoss()

    if args.cuda_graph and use_cuda:
        os.environ.setdefault("B200DP_FUSED_SINGLE", "1")    # graph capture needs the fused update
    optimizer = hvd.DistributedOptimizer(optimizer, named_parameters=model.named_parameters())

    model.to(_DEVICE)
    train_times = []

    hvd.broadcast_parameters(model.state_dict(), root_rank=0)

    def train_step(inputs, labels):
        pred = model(inputs)
        loss = loss_fn(pred.float(), labels)
        # Getting gradients w.r.t. parameters
        loss.backward()
        # Updating parameters
        optimizer.step()
        optimizer.zero_grad()
        return loss.detach()

    graphed = {}

    def train(epoch, device):
        loss = None
        for i, data in enumerate(train_loader):
            # move x and y to the device (no-op when the loader is device resident)
            inputs = data[0].to(_DEVICE, non_blocking=True)
            labels = data[1].to(_DEVICE, non_blocking=True)
            if args.cuda_graph and use_cuda and getattr(optimizer, "fused_engine", None) is not None:
                key = (tuple(inputs.shape), tuple(labels.shape))
                if key not in graphed and len(graphed) < 2:
                    from distributed_torch_horovod_gcp_b200.utils.graph import GraphedStep
                    graphed[key] = GraphedStep(train_step, [inputs, labels])
                loss = graphed[key](inputs, labels) if key in graphed else train_step(inputs, labels)
            else:
                loss = train_step(inputs, labels)
            if args.max_steps and i + 1 >= args.max_steps:
                break
        # write stats if running on main
        if device == 0:
            print(f"epoch: {epoch}, train_loss: {loss}", flush=True)

    def validate(epoch, device):
        test_loss = None
        for i, test_data in enumerate(test_loader):
            test_inputs, test_labels = test_data[0].to(_DEVICE), test_data[1].to(_DEVICE)
            test_pred = model(test_inputs)
            test_loss = loss_fn(test_pred.float(), test_labels)
        if device == 0:
            print(f"epoch: {epoch}, test_loss: {test_loss}", flush=True)

    # get statistics on the main node
    if device_number == 0:
        start_time = datetime.datetime.now()

    for epoch in range(epochs):
        epoch_start = datetime.datetime.now()
        train(epoch, device_number)
        if not args.no_validate:
            validate(epoch, device_number)
        epoch_end = datetime.datetime.now()
        epoch_time = (epoch_end - epoch_start).total_seconds()
        train_times.append(epoch_time)

    print(f"device: {hvd.rank()}, avg_time_per_epoch:{np.mean(train_times)}")
    if device_number == 0:
        end_time = datetime.datetime.now()
        total_time = (end_time - start_time).total_seconds() / 60
        print(f"total training time in minutes: {total_time}")
    hvd.shutdown()
