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
vit_b_16``, ``--dtype bf16``, ``--device cpu`` for the CPU/Gloo plumbing config, …), and the
GPT-2 causal language model on synthetic tokens (``--model gpt2|gpt-tiny``, ``--seq-len``).
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
    MinMaxScaler, StandardScaler, ensure_dataset, DeviceBatchLoader, SyntheticImageBatches, SyntheticTokenBatches)
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
                   help="synthetic image and GPT models only")
    p.add_argument("--seq-len", type=int, default=int(env("B200DP_SEQ_LEN", "0")),
                   help="GPT models: tokens per sequence (0 = the model's context)")
    p.add_argument("--no-validate", action="store_true")
    p.add_argument("--cuda-graph", action="store_true",
                   default=env("B200DP_CUDA_GRAPH", "0") == "1",
                   help="capture the whole training step (fwd+bwd+fused allreduce/update) in one "
                        "CUDA graph; H100-first answer for the launch-bound LSTM config")
    p.add_argument("--data", default=env("B200DP_DATA", "data_es.csv"))
    p.add_argument("--lstm-layers", type=int, default=int(env("B200DP_LSTM_LAYERS", "1")),
                   help="stacked LSTM layers of the lstm model (the reference uses 1)")
    p.add_argument("--bidirectional", action="store_true",
                   default=env("B200DP_BIDIRECTIONAL", "0") == "1",
                   help="bidirectional LSTM for the lstm model (the reference is unidirectional)")
    p.add_argument("--lstm-dropout", type=float, default=float(env("B200DP_LSTM_DROPOUT", "0")),
                   help="dropout probability between stacked LSTM layers (nn.LSTM dropout=; 0 = off, the "
                        "reference).  Like the reference, validation does not switch the model to eval mode, "
                        "so with P > 0 the printed test_loss is computed with dropout on")
    p.add_argument("--dropout", type=float, default=float(env("B200DP_DROPOUT", "0")),
                   help="dropout probability of the GPT and ViT models (GPT: embedding, attention and residual "
                        "dropout, as GPT-2's 0.1; ViT: token, attention and residual dropout; 0 = off)")
    p.add_argument("--clip-grad-norm", type=float, default=float(env("B200DP_CLIP_GRAD_NORM", "0")),
                   help="clip the averaged gradient by its global L2 norm to at most this value before "
                        "each update (DistributedOptimizer max_grad_norm=; 0 = off, the reference)")
    p.add_argument("--optimizer", default=env("B200DP_OPTIMIZER", "default"),
                   choices=["default", "lars", "lamb", "muon"],
                   help="image models: 'default' = SGD momentum 0.9, wd 1e-4 (the LSTM always uses Adam; "
                        "the GPT models AdamW, see gpt_optimizer); "
                        "'lars' / 'lamb' = hvd.LARS / hvd.LAMB with biases and norm-layer parameters in a "
                        "group with adaptive=False and no weight decay; "
                        "'muon' (GPT models only) = hvd.Muon on the blocks' matrices, AdamW on the rest "
                        "(see gpt_muon_optimizer)")
    p.add_argument("--sequence-parallel", action="store_true",
                   default=env("B200DP_SEQUENCE_PARALLEL", "0") == "1",
                   help="GPT models: split each sequence across the ranks (zigzag shards, sequence-parallel "
                        "attention) instead of giving each rank its own batch; every rank draws the same tokens "
                        "and keeps its shard, and the printed losses are the rank averages")
    sp_size = env("B200DP_SEQUENCE_PARALLEL_SIZE")
    p.add_argument("--sequence-parallel-size", type=int, default=int(sp_size) if sp_size else None, metavar="G",
                   help="with --sequence-parallel: split each sequence across a group of G ranks (G divides the "
                        "world size; groups are contiguous blocks of ranks) instead of the whole world; the ranks "
                        "of a group draw the same tokens and different groups different ones")
    args = p.parse_args(argv)
    if args.optimizer == "muon" and not is_gpt(args.model):
        p.error("--optimizer muon applies to the GPT models")
    if args.optimizer != "default" and args.model.lower() == "lstm":
        p.error("--optimizer lars|lamb applies to the image models")
    if not 0.0 <= args.dropout <= 1.0:
        p.error(f"--dropout must be in [0, 1], got {args.dropout}")
    if args.dropout and not (is_gpt(args.model) or is_vit(args.model)):
        p.error("--dropout applies to the GPT and ViT models (the LSTM has --lstm-dropout)")
    if args.sequence_parallel:
        if not is_gpt(args.model):
            p.error("--sequence-parallel applies to the GPT models")
        if args.dropout:
            p.error("--sequence-parallel does not support --dropout")
        if args.cuda_graph:
            p.error("--sequence-parallel cannot be combined with --cuda-graph: the sequence-parallel attention's "
                    "collectives are not captured in CUDA graphs")
    if args.sequence_parallel_size is not None:
        if not args.sequence_parallel:
            p.error("--sequence-parallel-size needs --sequence-parallel")
        from distributed_torch_horovod_gcp_b200._state import launch_size
        world = launch_size()
        if args.sequence_parallel_size < 1 or world % args.sequence_parallel_size:
            p.error(f"--sequence-parallel-size {args.sequence_parallel_size} does not divide the world size {world}")
    return args


def sp_split(args):
    """(group index, rank in the group, group size) of the sequence split: groups of --sequence-parallel-size
    contiguous ranks, or the whole world as one group."""
    G = args.sequence_parallel_size or hvd.size()
    return hvd.rank() // G, hvd.rank() % G, G


def image_optimizer(model, kind, lr):
    """The optimizer of the image models: SGD, or LARS / LAMB with 0/1-dim parameters (biases, BN / LN
    affine) excluded from weight decay and from the trust ratio."""
    if kind == "default":
        return torch.optim.SGD(model.parameters(), lr=lr, momentum=0.9, weight_decay=1e-4)
    groups = [{"params": [p for p in model.parameters() if p.dim() > 1]},
              {"params": [p for p in model.parameters() if p.dim() <= 1], "weight_decay": 0.0, "adaptive": False}]
    groups = [g for g in groups if g["params"]]
    if kind == "lars":
        return hvd.LARS(groups, lr=lr, momentum=0.9, weight_decay=1e-4)
    return hvd.LAMB(groups, lr=lr, weight_decay=0.01)


def is_gpt(name):
    return name.lower().replace("-", "").replace("_", "") in ("gpt2", "gpttiny")


def is_vit(name):
    return name.lower().replace("-", "").replace("_", "").startswith("vit")


def dropout_kw(args):
    """Model keyword arguments of ``--dropout`` (none at 0, so the models are built as without it)."""
    if not args.dropout:
        return {}
    if is_gpt(args.model):
        return {"dropout": args.dropout}
    return {"dropout": args.dropout, "attention_dropout": args.dropout}


def gpt_optimizer(model, lr):
    """The GPT-2 recipe: AdamW, betas (0.9, 0.95), weight decay 0.1 on matrices and embeddings (2 or more
    dimensions), none on biases and LayerNorm parameters."""
    groups = [{"params": [p for p in model.parameters() if p.dim() >= 2], "weight_decay": 0.1},
              {"params": [p for p in model.parameters() if p.dim() < 2], "weight_decay": 0.0}]
    return torch.optim.AdamW(groups, lr=lr, betas=(0.9, 0.95))


MUON_MATRICES = ("qkv.weight", "proj.weight", "fc1.weight", "fc2.weight")


def gpt_muon_optimizer(model, lr):
    """hvd.Muon on the transformer blocks' projection matrices (qkv, proj, fc1, fc2), with adjust_lr_fn
    "match_rms_adamw" so that gpt_optimizer's learning rate and weight decay carry over; the embeddings, biases
    and LayerNorm parameters keep gpt_optimizer's AdamW settings in use_muon=False groups."""
    named = list(model.named_parameters())
    muon = [p for n, p in named if n.startswith("layers.") and n.endswith(MUON_MATRICES)]
    ids = {id(p) for p in muon}
    rest = [p for _, p in named if id(p) not in ids]
    groups = [{"params": muon, "weight_decay": 0.1},
              {"params": [p for p in rest if p.dim() >= 2], "weight_decay": 0.1, "use_muon": False},
              {"params": [p for p in rest if p.dim() < 2], "weight_decay": 0.0, "use_muon": False}]
    return hvd.Muon([g for g in groups if g["params"]], lr=lr, betas=(0.9, 0.95),
                    adjust_lr_fn="match_rms_adamw")


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
                     n_layers=args.lstm_layers, bidirectional=args.bidirectional, device=_DEVICE,
                     dropout=args.lstm_dropout)
        optimizer = torch.optim.Adam(model.parameters(), lr=args.lr)
        loss_fn = nn.MSELoss(reduction="mean")
    elif is_gpt(args.model):
        sp_kw = {"sequence_parallel": True} if args.sequence_parallel else {}
        if args.sequence_parallel_size is not None:
            sp_kw["sequence_parallel_size"] = args.sequence_parallel_size
        model = build_model(args.model, **dropout_kw(args), **sp_kw).to(_DEVICE)
        if compute_dtype != torch.float32:
            model = model.to(compute_dtype)
        seq_len = args.seq_len or model.context
        # sequence parallelism: one batch per group (seeded by the group index), each rank keeps its zigzag shard
        # of every sequence
        sp_group, sp_rank, sp_world = sp_split(args) if args.sequence_parallel else (hvd.rank(), 0, 1)
        tokens = SyntheticTokenBatches(args.batch_size, seq_len, model.vocab, _DEVICE, seed=sp_group)

        def _next_tokens():
            inputs, labels = tokens.next()
            if not args.sequence_parallel:
                return inputs, labels
            from distributed_torch_horovod_gcp_b200.ops.seq_parallel import zigzag_shard
            shard = (lambda t: zigzag_shard(t, 1, sp_rank, sp_world))
            return shard(inputs), shard(labels.view(inputs.shape)).reshape(-1)

        class _TokenLoader:
            def __iter__(self_inner):
                for _ in range(args.steps_per_epoch):
                    yield _next_tokens()
        train_loader = _TokenLoader()
        test_loader = [_next_tokens()]
        lr = args.lr if args.lr != 1e-6 else 6e-4
        if args.optimizer == "default":
            optimizer = gpt_optimizer(model, lr)
        elif args.optimizer == "muon":
            optimizer = gpt_muon_optimizer(model, lr)
        else:
            optimizer = image_optimizer(model, args.optimizer, lr)
        loss_fn = nn.CrossEntropyLoss()
    else:
        small = args.model.lower().replace("-", "").replace("_", "") == "resnet18" and not use_cuda
        image_size = args.image_size or (32 if small else 224)
        num_classes = args.num_classes or (10 if small else 1000)
        kw = {"num_classes": num_classes}
        if "resnet" in args.model.lower():
            kw["small_input"] = image_size <= 64
        else:
            kw["image_size"] = image_size
        model = build_model(args.model, **kw, **dropout_kw(args)).to(_DEVICE)
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
        optimizer = image_optimizer(model, args.optimizer, lr)
        loss_fn = nn.CrossEntropyLoss()

    if args.cuda_graph and use_cuda:
        os.environ.setdefault("B200DP_FUSED_SINGLE", "1")    # graph capture needs the fused update
    optimizer = hvd.DistributedOptimizer(optimizer, named_parameters=model.named_parameters(),
                                         max_grad_norm=args.clip_grad_norm or None)

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
        if args.sequence_parallel:
            loss = hvd.allreduce(loss, average=True)      # each rank's loss is the mean over its own tokens
        # write stats if running on main
        if device == 0:
            print(f"epoch: {epoch}, train_loss: {loss}", flush=True)

    def validate(epoch, device):
        test_loss = None
        for i, test_data in enumerate(test_loader):
            test_inputs, test_labels = test_data[0].to(_DEVICE), test_data[1].to(_DEVICE)
            test_pred = model(test_inputs)
            test_loss = loss_fn(test_pred.float(), test_labels)
        if args.sequence_parallel:
            test_loss = hvd.allreduce(test_loss.detach(), average=True)
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
