"""Model zoo: the reference LSTM regressor plus the [DRIVER] benchmark families
(BASELINE.json configs): ResNet-18/50/152 and ViT-B/16, and the GPT-2 (124M) causal language model."""
from .gpt import GPT, gpt2, gpt_tiny  # noqa: F401
from .lstm import LSTM  # noqa: F401
from .resnet import ResNet, resnet18, resnet34, resnet50, resnet101, resnet152  # noqa: F401
from .vit import VisionTransformer, vit_b_16, vit_tiny  # noqa: F401


def build(name: str, **kw):
    name = name.lower().replace("-", "").replace("_", "")
    table = {"resnet18": resnet18, "resnet34": resnet34, "resnet50": resnet50,
             "resnet101": resnet101, "resnet152": resnet152, "vitb16": vit_b_16,
             "vittiny": vit_tiny, "gpt2": gpt2, "gpttiny": gpt_tiny}
    if name not in table:
        raise ValueError(f"unknown model {name!r}; have {sorted(table)} and 'lstm'")
    return table[name](**kw)
