"""TEST INFRASTRUCTURE ONLY.  The multiple-choice video QA graph (merlot_b200/video_mc.py) restated in fp32 autograd on top of
tests/multi_image_oracle.py (the joint encoder over F frames with img_mask) and tests/vcr_oracle.py (VCR's variables and
tower): one `mc_cls` tower over C candidates, softmax cross entropy over them, and the dropout hook that gives the oracle
the masks the kernels draw at the tower's two sites.
"""
from __future__ import annotations

import torch

from oracle import dropout_mask as DM
from tests import vcr_oracle as V

TOWER = "mc_cls"


def param_shapes(cfg: dict):
    """The VCR graph's model variables and one tower of the answer tower's shapes."""
    s = {k: v for k, v in V.param_shapes(cfg).items() if k.split("/")[0] not in V.TOWERS}
    s.update({k.replace("answer_cls/", f"{TOWER}/"): v for k, v in V.param_shapes(cfg).items() if k.startswith("answer_cls/")})
    return s


def init_params(cfg: dict, seed: int = 0, perturb: float = 0.0):
    """vcr_oracle.init_params with the answer tower's values under mc_cls and no rationale tower."""
    p = V.init_params(cfg, seed=seed, perturb=perturb)
    out = {k: v for k, v in p.items() if k.split("/")[0] not in V.TOWERS}
    out.update({k.replace("answer_cls/", f"{TOWER}/"): v for k, v in p.items() if k.startswith("answer_cls/")})
    return out


def mc_head_train(model, p, num_choices: int, dropout=None):
    """The tower on the oracle model's fp32 encoder_hidden_states['lang'][:, 0] -> logits [b, C]."""
    first = model.encoder_hidden_states["lang"][:, 0, :]  # [b*C, H], question-major
    x = first if dropout is None else dropout(("mc", "input"), first)
    from oracle import merlot_oracle as O
    h = O.dense(x, p, f"{TOWER}/classifier_mlp0", O.gelu)
    if dropout is not None:
        h = dropout(("mc", "hidden"), h)
    return O.dense(h, p, f"{TOWER}/classifier_mlp1").reshape(-1, num_choices)


def mc_loss(logits, target):
    """Mean softmax cross entropy over the candidates, and the accuracy."""
    return V.vcr_loss(logits, target)


def kernel_site(key) -> int:
    from merlot_b200 import modeling as M
    if key[0] != "mc":
        return DM.kernel_site(key)
    return {"input": M._SITE_MC_IN, "hidden": M._SITE_MC_HID}[key[1]]


def dropout_hook(seed: int, p: float, p_vit: float = None):
    """DM.dropout_hook(seed, p, p_vit) that also serves the tower's keys ("mc", "input" | "hidden") on its [b*C, N] rows."""
    base = DM.dropout_hook(seed, p, p_vit)

    def hook(key, x):
        if key[0] != "mc":
            return base(key, x)
        if p == 0.0:
            return x
        rows, N = x.shape
        keep = torch.from_numpy(DM.counter_dropout_keep(int(seed), kernel_site(key), rows, N, float(p)))
        return x * (keep.to(x.dtype) * float(DM.dropout_scale(p)))

    return hook
