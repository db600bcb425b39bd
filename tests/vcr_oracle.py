"""TEST INFRASTRUCTURE ONLY.  The VCR fine-tuning graph of downstream/vcr/modeling.py restated on top of the oracle
(oracle/merlot_oracle.py) in fp32 autograd, plus the dropout hook that gives the oracle the four classifier-tower masks the
CUDA path draws.  The existing oracle files are unchanged; this module only adds what the VCR step needs.

  * `param_shapes` / `init_params`: the variables of the VCR graph -- MerlotModel(mask_input=False) builds no language-only
    stack, no masking and no pretraining head (model/modeling.py:135-139 skipped), and the two towers of cls_head add
    `{answer,rationale}_cls/classifier_mlp{0,1}/{kernel,bias}` (downstream/vcr/modeling.py:86-121).
  * `vcr_cls_head_train`: cls_head (downstream/vcr/modeling.py:77-127).
  * `vcr_loss`: cls_loss + the accuracy metric (:13-20, :133-143).
  * `dropout_hook`: oracle/dropout_mask.dropout_hook extended with the keys ("vcr", tower, "input" | "hidden").
"""
from __future__ import annotations

import math

import torch

from oracle import dropout_mask as DM
from oracle import merlot_oracle as O

TOWERS = ("answer_cls", "rationale_cls")
_PRETRAIN_ONLY = ("langonly_embeddings/", "contrastive/", "lang_viz_temporal/", "viz_viz_temporal/", "lm_head/")


def param_shapes(cfg: dict):
    """Every trainable variable of the reference's VCR graph, at the reference's shapes."""
    s = {k: v for k, v in O.param_shapes(dict(cfg, num_lang_transformer_hidden_layers=0)).items()
         if not k.startswith(_PRETRAIN_ONLY)}
    H = cfg["hidden_size"]
    for tower in TOWERS:
        s[f"{tower}/classifier_mlp0/kernel"] = (H, H // 2)
        s[f"{tower}/classifier_mlp0/bias"] = (H // 2,)
        s[f"{tower}/classifier_mlp1/kernel"] = (H // 2, 1)
        s[f"{tower}/classifier_mlp1/bias"] = (1,)
    return s


def init_params(cfg: dict, seed: int = 0, perturb: float = 0.0):
    """O.init_params for the backbone; the towers get create_initializer kernels (truncated normal at initializer_range) and
    the classifier_mlp1 bias -log((1 - 0.25) / 0.25) (downstream/vcr/modeling.py:67-72,77)."""
    out = {k: v for k, v in O.init_params(dict(cfg, num_lang_transformer_hidden_layers=0), seed=seed, perturb=perturb).items()
           if not k.startswith(_PRETRAIN_ONLY)}
    g = torch.Generator().manual_seed(seed + 1)
    std = cfg.get("initializer_range", 0.02)
    for name, shape in param_shapes(cfg).items():
        if name.split("/")[0] not in TOWERS:
            continue
        if name.endswith("kernel"):
            t = O._trunc_normal(shape, std, g)
        elif name.endswith("classifier_mlp1/bias"):
            t = torch.full(shape, -math.log((1 - 0.25) / 0.25))
        else:
            t = torch.zeros(shape)
        if perturb > 0 and name.endswith("bias"):
            t = t + torch.randn(shape, generator=g) * perturb
        out[name] = t
    return out


def _tower(x, p, scope, dropout, tower):
    if dropout is not None:
        x = dropout(("vcr", tower, "input"), x)  # :87, :106
    h = O.dense(x, p, f"{scope}/classifier_mlp0", O.gelu)  # :88-94
    if dropout is not None:
        h = dropout(("vcr", tower, "hidden"), h)  # :95, :114
    return O.dense(h, p, f"{scope}/classifier_mlp1")  # :96-102


def vcr_cls_head_train(model, p, dropout=None):
    """cls_head (downstream/vcr/modeling.py:77-127) on the oracle model's fp32 encoder_hidden_states['lang'] -> [2b, 4]."""
    first = model.encoder_hidden_states["lang"][:, 0, :]  # :78
    H = first.shape[-1]
    first = first.reshape(-1, 2, 4, H)  # :79-80  [img_batch_size // 2, 2, num_texts, H]
    ans = first[:, 0].reshape(-1, H)  # :82-84
    rat = first[:, 1].reshape(-1, H)
    ans_logits = _tower(ans, p, "answer_cls", dropout, "answer").reshape(-1, 4)  # :103
    rat_logits = _tower(rat, p, "rationale_cls", dropout, "rationale").reshape(-1, 4)  # :122
    return torch.cat([ans_logits, rat_logits], 1).reshape(-1, 4)  # :124-125


def vcr_loss(logits_flat, target):
    """cls_loss (:133-143): sum of softmax cross entropy / img_batch_size; accuracy = mean of argmax == target (:13-20)."""
    per = O.raw_cross_entropy_with_logits(logits_flat, target.long())
    acc = (logits_flat.argmax(-1) == target.long()).float().mean()
    return per.sum() / logits_flat.shape[0], acc


def kernel_site(key) -> int:
    """The site of a classifier-tower dropout (merlot_b200/modeling.py _SITE_VCR_*); every other key as the oracle's."""
    from merlot_b200 import modeling as M
    if key[0] != "vcr":
        return DM.kernel_site(key)
    return {("answer", "input"): M._SITE_VCR_ANS_IN, ("answer", "hidden"): M._SITE_VCR_ANS_HID,
            ("rationale", "input"): M._SITE_VCR_RAT_IN, ("rationale", "hidden"): M._SITE_VCR_RAT_HID}[key[1:]]


def dropout_hook(seed: int, p: float, p_vit: float = None):
    """DM.dropout_hook(seed, p, p_vit) that also serves the four classifier-tower keys with hidden_dropout_prob p, on the
    tower's [4b, N] rows (question-major, candidate minor)."""
    base = DM.dropout_hook(seed, p, p_vit)

    def hook(key, x):
        if key[0] != "vcr":
            return base(key, x)
        if p == 0.0:
            return x
        rows, N = x.shape
        keep = torch.from_numpy(DM.counter_dropout_keep(int(seed), kernel_site(key), rows, N, float(p)))
        return x * (keep.to(x.dtype) * float(DM.dropout_scale(p)))

    return hook
