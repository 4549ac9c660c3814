"""Model zoo.  ``LinearModel``/``MLP2`` are portable; the ResNet / BERT / ViT
families are built from ``baton_b200.ops`` layers and import lazily."""
from .base import FederatedModule
from .linear import MLP2, LinearModel


def __getattr__(name):
    if name in ("ResNet", "resnet18", "resnet50"):
        from . import resnet
        return getattr(resnet, name)
    if name in ("BertConfig", "BertForSequenceClassification", "LoraConfig", "bert_base", "bert_tiny"):
        from . import bert
        return getattr(bert, name)
    if name in ("VisionTransformer", "vit_tiny", "vit_small"):
        from . import vit
        return getattr(vit, name)
    raise AttributeError(name)


__all__ = ["FederatedModule", "LinearModel", "MLP2", "resnet18", "resnet50", "bert_base", "vit_tiny", "vit_small"]
