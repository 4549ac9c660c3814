"""BERT-base sequence classifier on the sm_90a layers (benchmark configuration: the large
delta-reduce that stresses the NVLink roofline -- ~109.5 M parameters, 219 MB in bf16).

Standard post-LN encoder (embeddings -> 12 x [self-attention, FFN] -> pooler -> classifier) with
the usual parameter names (``bert.embeddings.word_embeddings.weight``,
``bert.encoder.layer.N.attention.self.query.weight`` ... are folded into one packed
``attention.qkv`` projection here for a single GEMM; ``load_hf_state_dict`` / ``hf_state_dict`` map a stock
Hugging-Face ``BertForSequenceClassification`` state_dict onto it and back, so HF checkpoints load and our
checkpoints stay loadable by HF -- tests/test_bert_hf_compat.py).  Every matmul is the wgmma
GEMM (GELU fused in the epilogue), attention is four strided-batched GEMMs + the softmax kernel on
the packed QKV buffer, LayerNorm fuses the residual add.  Dropout follows Hugging-Face's five positions with its
config names (``hidden_dropout_prob``, ``attention_probs_dropout_prob``, ``classifier_dropout``); the defaults are 0,
which runs exactly the kernels of a model without dropout.  The masks come from a counter (``data/dropout.py``), drawn
inside the fused attention, LayerNorm and softmax kernels; the trainers set the model's ``dropout_run`` before every
step, and nothing is dropped outside a training run or in eval mode.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import torch
from torch import nn

from ..data.dropout import DropoutRun, check_dropout
from ..ops import nn as bnn
from .base import FederatedModule


LORA_TARGETS = ("query", "key", "value", "attn_out", "ffn_in", "ffn_out")
LORA_RANKS = (8, 16, 32, 64)
# Hugging-Face module of each single-slice target, under bert.encoder.layer.N.
_LORA_HF = {"query": "attention.self.query", "key": "attention.self.key", "value": "attention.self.value",
            "attn_out": "attention.output.dense", "ffn_in": "intermediate.dense", "ffn_out": "output.dense"}


@dataclass(frozen=True)
class LoraConfig:
    """LoRA fine-tuning (PEFT's semantics): every targeted projection computes ``x W^T + b + s (x A^T) B^T`` with
    ``s = alpha / r``, ``A`` ``[r, in]`` from ``kaiming_uniform_(a=sqrt(5))`` and ``B`` ``[out, r]`` zero, so a fresh
    model computes what the base model does.  The base weights are frozen; the adapters and the classifier train.
    ``freeze_a``: FFA-LoRA -- ``A`` stays at its shared initial value, so the clients' mean of ``B`` is the mean of their
    products ``B A``."""
    r: int = 8
    alpha: float = 16.0
    targets: tuple = ("query", "value")
    freeze_a: bool = False

    def __post_init__(self):
        if isinstance(self.r, bool) or self.r not in LORA_RANKS:
            raise ValueError("LoRA: r must be one of {}, got {!r}".format(LORA_RANKS, self.r))
        if isinstance(self.alpha, bool) or not isinstance(self.alpha, (int, float)) or not self.alpha > 0:
            raise ValueError("LoRA: alpha must be a number > 0, got {!r}".format(self.alpha))
        t = (self.targets,) if isinstance(self.targets, str) else tuple(self.targets)
        if not t or len(set(t)) != len(t) or any(x not in LORA_TARGETS for x in t):
            raise ValueError("LoRA: targets must be distinct names from {}, got {!r}".format(LORA_TARGETS, self.targets))
        object.__setattr__(self, "targets", tuple(x for x in LORA_TARGETS if x in t))
        if not isinstance(self.freeze_a, bool):
            raise ValueError("LoRA: freeze_a must be a bool, got {!r}".format(self.freeze_a))

    @property
    def scale(self) -> float:
        return float(self.alpha) / self.r


@dataclass
class BertConfig:
    vocab_size: int = 30522
    hidden_size: int = 768
    num_hidden_layers: int = 12
    num_attention_heads: int = 12
    intermediate_size: int = 3072
    max_position_embeddings: int = 512
    type_vocab_size: int = 2
    layer_norm_eps: float = 1e-12
    num_labels: int = 2
    hidden_dropout_prob: float = 0.0
    attention_probs_dropout_prob: float = 0.0
    classifier_dropout: Optional[float] = None     # None: hidden_dropout_prob

    def __post_init__(self):
        check_dropout(self.hidden_dropout_prob, "hidden_dropout_prob")
        check_dropout(self.attention_probs_dropout_prob, "attention_probs_dropout_prob")
        if self.classifier_dropout is not None:
            check_dropout(self.classifier_dropout, "classifier_dropout")

    @property
    def classifier_p(self) -> float:
        return float(self.hidden_dropout_prob if self.classifier_dropout is None else self.classifier_dropout)


def _site(module: nn.Module, site: int, p: float):
    """``(run, site, p)`` when dropout site ``site`` drops in this call, else None."""
    run = module.dropout_run
    return (run, site, p) if p > 0.0 and module.training and run.active else None


class BertEmbeddings(nn.Module):
    def __init__(self, c: BertConfig, run: DropoutRun):
        super().__init__()
        self.dropout_run, self.p = run, float(c.hidden_dropout_prob)
        self.word_embeddings = bnn.Embedding(c.vocab_size, c.hidden_size)
        self.position_embeddings = bnn.Embedding(c.max_position_embeddings, c.hidden_size)
        self.token_type_embeddings = bnn.Embedding(c.type_vocab_size, c.hidden_size)
        self.LayerNorm = bnn.LayerNorm(c.hidden_size, c.layer_norm_eps)

    def forward(self, ids, pos_ids, type_ids):
        w = self.word_embeddings(ids)
        p = self.position_embeddings(pos_ids)
        t = self.token_type_embeddings(type_ids)
        drop = _site(self, 0, self.p)
        if drop is not None:
            drop = drop + (2,)                 # output dropout
        if w.is_cuda:
            pt = _Add.apply(p, t)
            return self.LayerNorm(w, pt) if drop is None else self.LayerNorm(w, pt, drop=drop)
        return self.LayerNorm(w + p + t) if drop is None else self.LayerNorm(w + p + t, drop=drop)


class _Add(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, b):
        from ..ops import functional as F
        return F.add(a, b)

    @staticmethod
    def backward(ctx, g):
        return g, g


class BertLayer(nn.Module):
    def __init__(self, c: BertConfig, run: DropoutRun, index: int):
        super().__init__()
        self.dropout_run, self.site = run, 1 + 3 * index        # sites: probabilities, attn_out, ffn_out
        self.p_attn, self.p_hidden = float(c.attention_probs_dropout_prob), float(c.hidden_dropout_prob)
        self.H, self.dh = c.num_attention_heads, c.hidden_size // c.num_attention_heads
        self.qkv = bnn.Linear(c.hidden_size, 3 * c.hidden_size)
        self.attn_out = bnn.Linear(c.hidden_size, c.hidden_size)
        self.attn_ln = bnn.LayerNorm(c.hidden_size, c.layer_norm_eps)
        self.ffn_in = bnn.Linear(c.hidden_size, c.intermediate_size, act="gelu")
        self.ffn_out = bnn.Linear(c.intermediate_size, c.hidden_size)
        self.ffn_ln = bnn.LayerNorm(c.hidden_size, c.layer_norm_eps)

    def forward(self, x, B, S, mask_bias=None):
        d_attn = _site(self, self.site, self.p_attn)
        if d_attn is None:
            a = bnn.attention(self.qkv(x), B, S, self.H, self.dh, mask_bias=mask_bias)
        else:
            a = bnn.attention(self.qkv(x), B, S, self.H, self.dh, mask_bias=mask_bias, drop=d_attn)
        d_out, d_ffn = _site(self, self.site + 1, self.p_hidden), _site(self, self.site + 2, self.p_hidden)
        if d_out is None:
            x = self.attn_ln(self.attn_out(a), x)
        else:
            x = self.attn_ln(self.attn_out(a), x, drop=d_out + (1,))        # input dropout
        if d_ffn is None:
            return self.ffn_ln(self.ffn_out(self.ffn_in(x)), x)
        return self.ffn_ln(self.ffn_out(self.ffn_in(x)), x, drop=d_ffn + (1,))


class BertForSequenceClassification(FederatedModule):
    name = "bert_base"
    loss_kind = "ce"
    default_lr = 0.01
    default_batch_size = 32
    head = "classifier"

    def __init__(self, config: Optional[BertConfig] = None, name: Optional[str] = None,
                 lora: Optional[LoraConfig] = None):
        super().__init__()
        if lora is not None and not isinstance(lora, LoraConfig):
            raise TypeError("lora= takes a LoraConfig, got {!r}".format(lora))
        self.config = c = config or BertConfig()
        if name:
            self.name = name
        self.dropout_run = DropoutRun()      # set by the trainers before every step (data/dropout.py)
        self.embeddings = BertEmbeddings(c, self.dropout_run)
        self.layers = nn.ModuleList([BertLayer(c, self.dropout_run, i) for i in range(c.num_hidden_layers)])
        self.pooler = bnn.Linear(c.hidden_size, c.hidden_size)
        self.classifier = bnn.Linear(c.hidden_size, c.num_labels, out_fp32=True)
        self._static = {}
        for m in self.modules():
            if isinstance(m, bnn.Linear):
                nn.init.normal_(m.weight, std=0.02)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)
        self.lora = lora
        if lora is not None:
            self._add_lora(lora)

    def _add_lora(self, lora: LoraConfig) -> None:
        """Adapters on the targeted projections of every layer, then everything but the adapters and the classifier
        frozen (``A`` too with ``freeze_a``)."""
        t = set(lora.targets)
        for layer in self.layers:
            if t & {"query", "key", "value"}:
                layer.qkv.add_lora(lora.r, lora.scale, tuple(n in t for n in ("query", "key", "value")))
            for name in ("attn_out", "ffn_in", "ffn_out"):
                if name in t:
                    getattr(layer, name).add_lora(lora.r, lora.scale, (True,))
        for n, p in self.named_parameters():
            train = n.startswith("classifier.") or n.endswith(".lora_B") or (n.endswith(".lora_A") and not lora.freeze_a)
            p.requires_grad_(train)

    @property
    def n_dropout_sites(self) -> int:
        return 2 + 3 * self.config.num_hidden_layers

    @property
    def has_dropout(self) -> bool:
        """True when some dropout probability is nonzero."""
        c = self.config
        return max(c.hidden_dropout_prob, c.attention_probs_dropout_prob, c.classifier_p) > 0.0

    def _ids(self, B, S, device):
        key = (B, S, str(device))
        if key not in self._static:
            pos = torch.arange(S, device=device).repeat(B)
            self._static[key] = (pos, torch.zeros(B * S, dtype=torch.long, device=device))
        return self._static[key]

    def forward(self, input_ids, attention_mask=None, token_type_ids=None):
        """``input_ids``: ``[B, S]`` int64 -> logits ``[B, num_labels]`` (fp32).  ``attention_mask`` (``[B, S]``, 1 =
        attend, 0 = padding) and ``token_type_ids`` follow the Hugging-Face call convention; without a mask the
        attention core takes its unmasked fast path."""
        B, S = input_ids.shape
        pos, typ = self._ids(B, S, input_ids.device)
        if token_type_ids is not None:
            typ = token_type_ids.reshape(-1)
        mask_bias = None
        if attention_mask is not None:
            mask_bias = (1.0 - attention_mask.to(torch.float32)) * -30000.0      # additive, finite in bf16
        x = self.embeddings(input_ids, pos, typ)
        for layer in self.layers:
            x = layer(x, B, S, mask_bias)
        first = x.view(B, S, -1)[:, 0].contiguous()
        pooled = torch.tanh(self.pooler(first).float())
        if pooled.is_cuda:
            pooled = pooled.to(torch.bfloat16)
        drop = _site(self, self.n_dropout_sites - 1, self.config.classifier_p)
        if drop is not None:
            pooled = bnn.dropout(pooled, *drop)
        return self.classifier(pooled)


    # ------------------------------------------------------------------ Hugging-Face checkpoint compatibility
    _HF_LAYER = (("attention.output.dense", "attn_out"), ("attention.output.LayerNorm", "attn_ln"),
                 ("intermediate.dense", "ffn_in"), ("output.dense", "ffn_out"), ("output.LayerNorm", "ffn_ln"))

    @torch.no_grad()
    def load_hf_state_dict(self, hf_state: dict, strict: bool = True) -> None:
        """Load a stock ``transformers.BertForSequenceClassification`` ``state_dict``: the separate query / key /
        value projections are concatenated (rows ``[q; k; v]``) into the packed ``qkv`` GEMM, everything else is a
        rename.  Note: this model uses the tanh GELU (``hidden_act="gelu_pytorch_tanh"`` in HF terms)."""
        own = {}
        sd = dict(hf_state)
        for k in ("word_embeddings", "position_embeddings", "token_type_embeddings"):
            own["embeddings.{}.weight".format(k)] = sd.pop("bert.embeddings.{}.weight".format(k))
        for p in ("weight", "bias"):
            own["embeddings.LayerNorm." + p] = sd.pop("bert.embeddings.LayerNorm." + p)
        for i in range(self.config.num_hidden_layers):
            hf, me = "bert.encoder.layer.{}.".format(i), "layers.{}.".format(i)
            for p in ("weight", "bias"):
                own[me + "qkv." + p] = torch.cat([sd.pop(hf + "attention.self.{}.{}".format(n, p))
                                                  for n in ("query", "key", "value")], dim=0)
                for a, b in self._HF_LAYER:
                    own[me + b + "." + p] = sd.pop(hf + a + "." + p)
        for p in ("weight", "bias"):
            own["pooler." + p] = sd.pop("bert.pooler.dense." + p)
            own["classifier." + p] = sd.pop("classifier." + p)
        sd.pop("bert.embeddings.position_ids", None)
        sd.pop("bert.embeddings.token_type_ids", None)
        if strict and sd:
            raise KeyError("unexpected Hugging-Face keys: {}".format(sorted(sd)[:5]))
        missing, unexpected = self.load_state_dict(own, strict=False)     # a LoRA model keeps its adapters
        missing = [k for k in missing if not k.endswith((".lora_A", ".lora_B"))]
        if strict and (missing or unexpected):
            raise KeyError("state_dict mismatch: missing {}, unexpected {}".format(missing[:5], unexpected[:5]))
        arena = getattr(self, "_arena", None)
        if arena is not None:
            arena.commit_global()

    def hf_state_dict(self) -> dict:
        """Inverse of :meth:`load_hf_state_dict`: a ``state_dict`` a stock Hugging-Face model loads with ``strict=True``."""
        own = {k: v.detach() for k, v in self.state_dict().items()}
        D = self.config.hidden_size
        out = {}
        for k in ("word_embeddings", "position_embeddings", "token_type_embeddings"):
            out["bert.embeddings.{}.weight".format(k)] = own["embeddings.{}.weight".format(k)]
        for p in ("weight", "bias"):
            out["bert.embeddings.LayerNorm." + p] = own["embeddings.LayerNorm." + p]
        for i in range(self.config.num_hidden_layers):
            hf, me = "bert.encoder.layer.{}.".format(i), "layers.{}.".format(i)
            for p in ("weight", "bias"):
                q = own[me + "qkv." + p]
                for j, n in enumerate(("query", "key", "value")):
                    out[hf + "attention.self.{}.{}".format(n, p)] = q[j * D:(j + 1) * D].clone()
                for a, b in self._HF_LAYER:
                    out[hf + a + "." + p] = own[me + b + "." + p]
        for p in ("weight", "bias"):
            out["bert.pooler.dense." + p] = own["pooler." + p]
            out["classifier." + p] = own["classifier." + p]
        return out


    # ------------------------------------------------------------------ LoRA adapters under Hugging-Face names
    def _lora_modules(self):
        """``(HF module prefix, layer, rank block, slice)`` of every adapter: the packed ``qkv`` layer holds one rank
        block per targeted slice."""
        if self.lora is None:
            raise RuntimeError("this model has no LoRA adapters (build it with lora=LoraConfig(...))")
        out = []
        for i, layer in enumerate(self.layers):
            hf = "bert.encoder.layer.{}.".format(i)
            for mod, names in ((layer.qkv, ("query", "key", "value")), (layer.attn_out, ("attn_out",)),
                               (layer.ffn_in, ("ffn_in",)), (layer.ffn_out, ("ffn_out",))):
                if getattr(mod, "lora_cfg", None) is None:
                    continue
                slot = mod.lora_cfg[2]
                for j, n in enumerate(names):
                    if slot[j] >= 0:
                        out.append((hf + _LORA_HF[n], mod, slot[j], j))
        return out

    @torch.no_grad()
    def lora_state_dict(self) -> dict:
        """The trainable entries -- every adapter's ``lora_A.weight`` ``[r, in]`` and ``lora_B.weight`` ``[out, r]``
        under its Hugging-Face module name, and ``classifier.weight`` / ``.bias`` -- as fp32 copies."""
        r = self.lora.r
        out = {}
        for name, mod, t, _ in self._lora_modules():
            ds = mod.lora_cfg[3]
            out[name + ".lora_A.weight"] = mod.lora_A[t * r:(t + 1) * r].detach().clone()
            out[name + ".lora_B.weight"] = mod.lora_B[t * ds:(t + 1) * ds].detach().clone()
        for p in ("weight", "bias"):
            out["classifier." + p] = getattr(self.classifier, p).detach().clone()
        return out

    @torch.no_grad()
    def load_lora_state_dict(self, state: dict) -> None:
        """Inverse of :meth:`lora_state_dict`; every key must be present and no other."""
        own = self.lora_state_dict()
        if set(state) != set(own):
            raise KeyError("LoRA state_dict keys differ: missing {}, unexpected {}".format(
                sorted(set(own) - set(state))[:5], sorted(set(state) - set(own))[:5]))
        r = self.lora.r
        for name, mod, t, _ in self._lora_modules():
            ds = mod.lora_cfg[3]
            mod.lora_A[t * r:(t + 1) * r].copy_(state[name + ".lora_A.weight"])
            mod.lora_B[t * ds:(t + 1) * ds].copy_(state[name + ".lora_B.weight"])
        for p in ("weight", "bias"):
            getattr(self.classifier, p).copy_(state["classifier." + p])
        arena = getattr(self, "_arena", None)
        if arena is not None:
            arena.commit_global()

    @torch.no_grad()
    def merged_hf_state_dict(self) -> dict:
        """A stock Hugging-Face ``state_dict`` (as :meth:`hf_state_dict`) with every adapter merged, ``W + s B A``
        computed in float64 and rounded to fp32 once: it loads with ``strict=True`` into a model without LoRA."""
        out = self.hf_state_dict()
        s, r = self.lora.scale, self.lora.r
        for name, mod, t, _ in self._lora_modules():
            ds = mod.lora_cfg[3]
            a = mod.lora_A[t * r:(t + 1) * r].double()
            b = mod.lora_B[t * ds:(t + 1) * ds].double()
            w = out[name + ".weight"]
            out[name + ".weight"] = (w.double() + s * (b @ a).to(w.device)).float()
        return out


def bert_base(num_labels: int = 2, lora: Optional[LoraConfig] = None, **kw) -> BertForSequenceClassification:
    return BertForSequenceClassification(BertConfig(num_labels=num_labels, **kw), lora=lora)


def bert_tiny(num_labels: int = 2, lora: Optional[LoraConfig] = None) -> BertForSequenceClassification:
    """2-layer, 128-wide model for tests."""
    return BertForSequenceClassification(BertConfig(vocab_size=1024, hidden_size=128, num_hidden_layers=2,
                                                    num_attention_heads=2, intermediate_size=512,
                                                    max_position_embeddings=128, num_labels=num_labels), name="bert_tiny",
                                         lora=lora)
