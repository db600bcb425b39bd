"""The pretraining gradient one loss at a time, in float64: the oracle's gradient of each loss alone (and of their sum), the
comparisons the per-loss tests make (per-tensor error, exact zero pattern, per-row checks of the gathered tables), the bars
those comparisons use, and wrong-path variants of the oracle that the bars must reject.

A test of the summed gradient cannot see a path that carries a small share of a tensor's gradient (the MLM loss gives the
vision tower well under 1% of its gradient at the tiny config), so every path is compared against the gradient of its own
loss.  Only tests/ import this module."""
from __future__ import annotations

from typing import Dict, Optional

import torch

from oracle import merlot_oracle as O

LOSSES = ("mlm", "ctr", "tmp")
SUBSETS = {"mlm": ("mlm",), "ctr": ("ctr",), "tmp": ("tmp",), "all": LOSSES}

# Bars, each about 2x the worst error measured on an H100 80GB HBM3 at a 700 W power limit for that loss and case (the GPU
# backward is repeatable to ~3e-7, so one measurement stands for every run).  tests/test_gpu_loss_paths.py writes the full
# table to its JSON report.  Measured worst tensor / median over the tensors the oracle gives a gradient:
#
#   case   mlm               ctr               tmp               all
#   eval   8.8e-3 / 5.3e-3   2.7e-2 / 1.7e-2   1.2e-2 / 6.2e-3   2.2e-2 / 1.1e-2
#   train  8.4e-3 / 6.1e-3   1.8e-2 / 1.3e-2   1.2e-2 / 6.5e-3   1.8e-2 / 1.0e-2
#   long   8.9e-3 / 5.6e-3   1.6e-2 / 9.6e-3   8.4e-3 / 3.1e-3   1.5e-2 / 9.0e-3
#
# The contrastive loss is the least exact: its temperature (0.05) multiplies the bf16 rounding of the features twenty-fold
# in the logits, and every gradient it sends back carries that.
#   tensor: relative Frobenius error of one parameter gradient against the float64 oracle's gradient of the same loss.
BARS = {
    "eval": {"mlm": 2e-2, "ctr": 6e-2, "tmp": 2.5e-2, "all": 4.5e-2},
    "train": {"mlm": 2e-2, "ctr": 4e-2, "tmp": 2.5e-2, "all": 4e-2},
    "long": {"mlm": 2e-2, "ctr": 3.5e-2, "tmp": 2e-2, "all": 3.5e-2},
}
#   row: relative error of one row of a gathered / scattered table (ROW_TABLES) on its own.  Measured worst row:
#   mlm 6.7e-3 / 8.8e-3 / 8.8e-3, tmp 8.2e-3 / 8.9e-3 / 6.2e-3 (eval / train / long); under the contrastive loss the
#   language-only position rows of the pooled first tokens, 5.4e-2 / 5.3e-2 / 5.6e-2, each the gradient of one feature row.
ROW_BARS = {
    "eval": {"mlm": 1.5e-2, "ctr": 0.11, "tmp": 2e-2, "all": 0.11},
    "train": {"mlm": 2e-2, "ctr": 0.11, "tmp": 2e-2, "all": 0.11},
    "long": {"mlm": 2e-2, "ctr": 0.12, "tmp": 1.5e-2, "all": 0.12},
}
# Sum check: the three per-loss GPU gradients summed against the GPU gradient of all three.  bwd.d_yj is bf16, so the MLM and
# temporal terms meet there rounded once when they run together and twice when they run apart: the bar is at bf16 level.
# Measured worst tensor 7.6e-3 / 6.3e-3 / 4.9e-3 (eval / train / long).
SUM_BAR = 1.5e-2
# Side stream: the language-only backward on its side stream against the same backward on one stream, and two default runs
# against each other (fp32 atomic adds in another order), relative error per tensor.  Measured worst over two runs 3.8e-7
# (one stream) and 4.5e-7 (repeat); the bar is the floor of 1e-6.
SIDE_BAR = 1e-6
# The old whole-step bar of tests/test_gpu_model.py (the gradient of the sum of the three losses, per tensor).
SUMMED_STEP_BAR = 4e-2

# Tables fed through a gather or scatter: the reference name and how its rows are laid out.
ROW_TABLES = (
    "word_embeddings/word_embeddings",
    "position_embeddings/position_embeddings",
    "langonly_embeddings/position_embeddings",
    "vision_backbone/vision_transformer/pos_embs/pos_embs",
    "vision_backbone/vision_transformer/pos_embs/cls_emb",
    "vision_backbone/final_pe/pos_embs",
    "vision_backbone/final_pe/cls_emb",
    "vision_backbone/img_idx_pe",
)


def is_shift_invariant(name: str) -> bool:
    """Softmax is invariant to a shift of every score of a row, and the key bias shifts them so: its gradient is zero up to
    rounding in the oracle and on the GPU, so neither its error nor its zero pattern says anything."""
    return name.endswith("key_layer/bias")


def rows_of(name: str, t: torch.Tensor) -> torch.Tensor:
    """The table as [rows, H]: [1, 64, 64, H] position grids as 4096 rows (row = i * 64 + j), [1, n, H] cls tables as n."""
    return t.reshape(-1, t.shape[-1])


def rel(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-300))


def tiny_params(cfg: dict, seed: int = 1) -> Dict[str, torch.Tensor]:
    """The parameters of tests/test_gpu_model.py's build() in float64: the initial values are drawn in float32, and GEMM
    operands (kernels, the word embedding) are rounded to bf16 as the GPU's compute copies are, so both sides hold the very
    same numbers."""
    p = O.init_params(cfg, seed=seed, dtype=torch.float64, perturb=0.05)
    return {k: (v.bfloat16().double() if (k.endswith("kernel") or k.endswith("word_embeddings")) else v) for k, v in p.items()}


class PathOracle(O.MerlotOracle):
    """MerlotOracle with one gradient path cut or misrouted (`variant`), to show that the per-loss bars reject such a path:
      None           the oracle itself;
      "mlm_no_viz"   the MLM loss reads a joint encoder whose vision rows are detached (MLM never reaches the vision tower);
      "tmp_swap"     the lang_viz temporal head reads (viz, lang) pairs in place of (lang, viz);
      "ctr_no_lang"  the contrastive loss reads the language-only features detached (the language-only tower gets nothing)."""

    VARIANTS = (None, "mlm_no_viz", "tmp_swap", "ctr_no_lang")

    def __init__(self, config, params, image, input_ids, variant: Optional[str] = None, dropout=None, **kw):
        if variant not in self.VARIANTS:
            raise ValueError(f"unknown variant {variant!r}")
        self.variant, self._dropout = variant, dropout
        super().__init__(config, params, image, input_ids, dropout=dropout, **kw)
        if variant == "ctr_no_lang":
            self.lang_trg_h = self.lang_trg_h.detach()

    def mask_loss(self):
        if self.variant != "mlm_no_viz":
            return super().mask_loss()
        assert not self.config.get("disable_pairwise_lang_attn", False)
        viz, lang = self.encoder_pieces
        enc_in = torch.cat([viz["x"].detach(), lang["x"]], 1)
        valid = torch.cat([viz["is_valid"], lang["is_valid"]], 1)
        mask = (valid[:, None] & valid[:, :, None]).to(enc_in.dtype)
        h = O.transformer(enc_in, mask, self.p, "encoder", self.config["num_hidden_layers"], self.config["num_attention_heads"],
                          dropout=O._scoped(self._dropout, "joint"))["hidden_state"]
        kept = self.encoder_hidden_states
        self.encoder_hidden_states = {"viz": h[:, :viz["end"]], "lang": h[:, lang["start"]:]}
        try:
            return super().mask_loss()
        finally:
            self.encoder_hidden_states = kept

    def allpairs_temporal_logits(self, xa, xb, scope_name):
        if self.variant == "tmp_swap" and scope_name == "lang_viz_temporal":
            xa, xb = xb, xa
        return super().allpairs_temporal_logits(xa, xb, scope_name)


def oracle_losses(om: O.MerlotOracle, shuf, vid) -> Dict[str, torch.Tensor]:
    """The three losses of model_fn (model/modeling.py:700-713), each on its own."""
    out = {"mlm": om.mask_loss()[0], "ctr": om.contrastive_loss()[0]}
    out["tmp"] = om.temporal_loss(shuf, vid)[0]
    return out


def oracle_grads(cfg, params, image, ids, shuf, vid, masks, dropout=None, variant=None) -> Dict[str, Dict[str, torch.Tensor]]:
    """{subset: {name: float64 gradient}} for every subset of SUBSETS, on one float64 oracle graph fed the GPU-chosen `masks`
    ({'masked_ids', 'masked_idx'}).  A variable the subset never reaches gets an all-zero gradient.  'all' is differentiated
    as the sum itself, not summed from the parts."""
    leaf = {k: v.detach().double().clone().requires_grad_(True) for k, v in params.items()}
    om = PathOracle(cfg, leaf, image.double(), ids, variant=variant, dropout=dropout, mask_input=True, shuffled_idx_img=shuf,
                    mask_override=masks)
    losses = oracle_losses(om, shuf, vid)
    names = list(leaf)
    out = {}
    for sub, parts in SUBSETS.items():
        total = sum(losses[p] for p in parts)
        gs = torch.autograd.grad(total, [leaf[k] for k in names], retain_graph=True, allow_unused=True)
        out[sub] = {k: (torch.zeros_like(leaf[k]) if g is None else g.detach()) for k, g in zip(names, gs)}
    return out


def tensor_errors(got: Dict[str, torch.Tensor], ref: Dict[str, torch.Tensor]) -> Dict[str, float]:
    """Relative Frobenius error of every gradient the reference gives a non-zero value (the key biases excepted)."""
    return {k: rel(got[k], r) for k, r in ref.items() if not is_shift_invariant(k) and float(r.abs().max()) > 0}


def zero_pattern_violations(got: Dict[str, torch.Tensor], ref: Dict[str, torch.Tensor]) -> Dict[str, str]:
    """Names whose zero pattern differs from the reference's: an element the reference holds exactly zero that is not zero
    in `got`, or a tensor the reference gives a non-zero gradient that `got` leaves entirely zero.  A key bias is held to
    its pattern only where the reference leaves it entirely zero."""
    bad = {}
    for k, r in ref.items():
        g = got[k].double()
        if is_shift_invariant(k) and float(r.abs().max()) > 0:  # rounding noise, exactly zero here and there on either side
            continue
        stray = int(((r == 0) & (g != 0)).sum())
        if stray:
            bad[k] = f"{stray} elements non-zero where the oracle is exactly zero (max |g| {float(g[r == 0].abs().max()):.3e})"
        elif float(r.abs().max()) > 0 and float(g.abs().max()) == 0:
            bad[k] = "all zero where the oracle is not"
    return bad


def nonzero_rows(name: str, t: torch.Tensor) -> set:
    return set(torch.nonzero(rows_of(name, t).abs().amax(1) > 0).reshape(-1).tolist())


def row_report(name: str, got: torch.Tensor, ref: torch.Tensor) -> dict:
    """The rows of table `name` with a non-zero gradient in `got` and in `ref`, and the relative error of every row the
    reference gives a gradient: {'extra': rows only in got, 'missing': rows only in ref, 'worst': (row, error), 'n': rows}."""
    rg, rr = nonzero_rows(name, got), nonzero_rows(name, ref)
    G, R = rows_of(name, got).double(), rows_of(name, ref)
    errs = {i: float((G[i] - R[i]).norm() / R[i].norm()) for i in sorted(rr)}
    worst = max(errs.items(), key=lambda kv: kv[1]) if errs else (None, 0.0)
    return {"extra": sorted(rg - rr), "missing": sorted(rr - rg), "worst": worst, "n": len(rr)}


def move_row(grads: Dict[str, torch.Tensor], name: str, row: int) -> Dict[str, torch.Tensor]:
    """A copy of `grads` with row `row` of table `name` added to row `row + 1` and cleared: one gradient row misrouted."""
    out = dict(grads)
    t = rows_of(name, grads[name]).clone()
    t[row + 1] += t[row]
    t[row] = 0
    out[name] = t.reshape(grads[name].shape)
    return out


def summary(errs: Dict[str, float]) -> dict:
    """Worst tensor and median of a {name: error} table."""
    if not errs:
        return {"worst": None, "worst_err": 0.0, "median": 0.0, "n": 0}
    k = max(errs, key=errs.get)
    v = sorted(errs.values())
    med = v[len(v) // 2] if len(v) % 2 else 0.5 * (v[len(v) // 2 - 1] + v[len(v) // 2])
    return {"worst": k, "worst_err": errs[k], "median": med, "n": len(v)}
