"""The pretraining backward one loss at a time (pytest -m gpu): MerlotModel.backward after only the MLM, only the contrastive,
only the temporal head, and all three, each against the float64 oracle's gradient of that loss alone -- every parameter
tensor, the exact zero pattern, the rows of the gathered / scattered tables, the sum of the three, and the language-only
backward on its side stream against the same backward on one stream.

The summed-loss parity of tests/test_gpu_model.py cannot see a path that carries a small share of a tensor's gradient (the MLM
loss gives the vision tower under 1% of its gradient here, tests/test_loss_paths_host.py), nor one misrouted row of an
embedding table.  Bars and their basis are in tests/loss_paths_oracle.py.  Every measured error goes into a JSON report:
$MERLOT_LOSS_PATHS_REPORT if set, else a fresh file under the temporary directory (its path is printed)."""
import json
import os
import tempfile

import pytest
import torch

from oracle import merlot_oracle as O
from tests import loss_paths_oracle as LP
from tests.test_gpu_model import build, synth

pytestmark = pytest.mark.gpu
DEV = "cuda"
_report = {"path": None, "data": {}}
_cache = {}


def record(section, payload):
    if _report["path"] is None:
        _report["path"] = os.environ.get("MERLOT_LOSS_PATHS_REPORT") or os.path.join(
            tempfile.mkdtemp(prefix="merlot_loss_paths_"), "loss_paths.json")
        print(f"loss-path report: {_report['path']}")
    _report["data"][section] = payload
    with open(_report["path"], "w") as f:
        json.dump(_report["data"], f, indent=1, sort_keys=True)


def _case_setup(case, tiny_cfg):
    """eval / train: the inputs of test_pretrain_step_parity(_training_mode); long: those of
    test_pretrain_step_parity_long_sequence (L = 640, Sj = 696: attention backward with atomic dQ), in training mode."""
    from oracle import dropout_mask as DM
    if case == "eval":
        return dict(cfg=dict(tiny_cfg), training=False, seed=0, hook=None, batch=2, nc=4, Lc=16)
    if case == "train":
        seed = 2 ** 32 + 77
        return dict(cfg=dict(tiny_cfg, hidden_dropout_prob=0.1, vit_hidden_dropout_prob=0.2), training=True, seed=seed,
                    hook=DM.dropout_hook(seed, 0.1, 0.2), batch=2, nc=4, Lc=16)
    assert case == "long"
    seed = 2 ** 32 + 78
    return dict(cfg=dict(tiny_cfg, num_chunks_in_group=8, max_position_embeddings=1024, hidden_dropout_prob=0.1,
                         vit_hidden_dropout_prob=0.2), training=True, seed=seed, hook=DM.dropout_hook(seed, 0.1, 0.2),
                batch=1, nc=8, Lc=80)


class _Runner:
    """One case's inputs on the GPU: a fresh MerlotModel per run, on freshly zeroed gradients, calling only the chosen heads."""

    def __init__(self, case, tiny_cfg):
        s = _case_setup(case, tiny_cfg)
        self.cfg, self.training, self.seed, self.hook = s["cfg"], s["training"], s["seed"], s["hook"]
        self.image, self.ids, self.shuf, self.vid = synth(self.cfg, s["batch"], s["nc"], s["Lc"], 64, 96, 0)
        params32, self.store, _ = build(self.cfg)
        self.params = {k: v.double() for k, v in params32.items()}  # the same numbers (drawn in fp32, GEMM operands bf16)
        assert all(torch.equal(self.params[k], v) for k, v in LP.tiny_params(self.cfg).items())
        B, Lj = s["batch"] * s["nc"] // self.cfg["num_chunks_in_group"], s["Lc"] * self.cfg["num_chunks_in_group"]
        draws = O.make_mask_draws(B, Lj, int(Lj * 0.2), self.cfg["vocab_size"], seed=5)
        m = self._model(mask_draws=draws)
        self.masks = {"masked_ids": m.lang_mask_info["masked_ids"].cpu().reshape(B, Lj),
                      "masked_idx": m.lang_mask_info["masked_idx"].cpu()}

    def _model(self, **kw):
        from merlot_b200.modeling import MerlotModel
        return MerlotModel(self.cfg, is_training=self.training, use_tpu=False, image=self.image.to(DEV),
                           input_ids=self.ids.to(DEV), mask_input=True, shuffled_idx_img=self.shuf.to(DEV), params=self.store,
                           save_for_backward=True, dropout_seed=self.seed, **kw)

    def grads(self, subset):
        m = self._model(mask_override=self.masks)
        parts = LP.SUBSETS[subset]
        if "mlm" in parts:
            m.mask_loss()
        if "ctr" in parts:
            m.contrastive_loss()
        if "tmp" in parts:
            m.temporal_loss(self.shuf.to(DEV), self.vid.to(DEV))
        self.store.g.zero_()
        m.backward()
        torch.cuda.synchronize()
        g = {k: v.double() for k, v in self.store.to_tf_dict("g").items()}
        self.store.g.zero_()
        return g

    def oracle(self, variant=None):
        return LP.oracle_grads(self.cfg, self.params, self.image, self.ids, self.shuf, self.vid, self.masks, dropout=self.hook,
                               variant=variant)


def _results(case, tiny_cfg):
    """GPU and oracle gradients of every subset of one case, computed once per module."""
    if case not in _cache:
        r = _Runner(case, tiny_cfg)
        _cache[case] = (r, {s: r.grads(s) for s in LP.SUBSETS}, r.oracle())
    return _cache[case]


CASES = ("eval", "train", "long")


@pytest.mark.parametrize("case", CASES)
def test_per_loss_gradient_parity(case, tiny_cfg):
    """Every parameter gradient of each loss alone against the float64 oracle's gradient of that loss alone.  Bar: about 2x
    the worst tensor measured on the H100 for that loss and case (loss_paths_oracle.BARS)."""
    _, gpu, ref = _results(case, tiny_cfg)
    table, bad = {}, []
    for sub in LP.SUBSETS:
        errs = LP.tensor_errors(gpu[sub], ref[sub])
        table[sub] = dict(LP.summary(errs), bar=LP.BARS[case][sub], tensors=errs)
        bad += [(sub, k, e) for k, e in errs.items() if not e <= LP.BARS[case][sub]]
    record(f"{case}/tensors", table)
    assert not bad, sorted(bad, key=lambda t: -t[2])[:8]


@pytest.mark.parametrize("case", CASES)
def test_per_loss_zero_pattern(case, tiny_cfg):
    """Where the float64 oracle's gradient of a loss is exactly zero the GPU's is exactly zero, element by element (e.g. lm_head
    and contrastive under the temporal loss, the joint position table under the contrastive loss); where the oracle's is not,
    the GPU's is not."""
    _, gpu, ref = _results(case, tiny_cfg)
    bad = {sub: LP.zero_pattern_violations(gpu[sub], ref[sub]) for sub in LP.SUBSETS}
    zero = {sub: sorted(k for k, v in ref[sub].items() if float(v.abs().max()) == 0) for sub in LP.SUBSETS}
    record(f"{case}/zero_pattern", {"violations": bad, "oracle_zero_tensors": zero})
    # each single loss leaves variables untouched: the other heads, and the joint encoder's inputs under the contrastive loss,
    # whose features never pass through it (encoder/ itself is shared with the language-only stack and is reached)
    assert {"lm_head/output_bias", "contrastive/lang_proj/kernel"} <= set(zero["tmp"])
    assert {"lang_viz_temporal/logits/kernel", "viz_viz_temporal/intermediate/kernel"} <= set(zero["mlm"])
    assert "position_embeddings/position_embeddings" in zero["ctr"]
    assert "encoder/layer00/query_layer/kernel" not in zero["ctr"] and not zero["all"]
    assert not any(bad.values()), bad


@pytest.mark.parametrize("case", CASES)
def test_per_loss_table_rows(case, tiny_cfg):
    """The gathered / scattered tables row by row: the rows with a non-zero gradient are exactly the oracle's (word rows of the
    original ids under the contrastive loss, of the masked ids under the temporal loss, every row under MLM; the position
    rows where some sequence has a valid token; the h1 x w1 and h2 x w2 grids; the img_idx_pe rows of shuffled_idx_img; the
    cls rows: tests/test_loss_paths_host.py derives the oracle's sets from the inputs), and
    each of them is within a per-row bar (loss_paths_oracle.ROW_BARS: about 2x the worst row measured on the H100)."""
    _, gpu, ref = _results(case, tiny_cfg)
    out, bad = {}, []
    for sub in LP.SUBSETS:
        for name in LP.ROW_TABLES:
            r = LP.row_report(name, gpu[sub][name], ref[sub][name])
            out[f"{sub}/{name}"] = r
            if r["extra"] or r["missing"] or not r["worst"][1] <= LP.ROW_BARS[case][sub]:
                bad.append((sub, name, r))
    record(f"{case}/rows", out)
    assert not bad, bad[:4]


@pytest.mark.parametrize("case", CASES)
def test_per_loss_gradients_sum_to_the_step(case, tiny_cfg):
    """The three per-loss GPU gradients, summed, match the GPU gradient of all three.  bwd.d_yj is bf16, so the MLM and
    temporal terms are rounded once together and twice apart: the bar (loss_paths_oracle.SUM_BAR) is at bf16 level.  A buffer
    zeroed on some paths only, or a result that depends on which other heads ran, gives errors of order one."""
    _, gpu, _ = _results(case, tiny_cfg)
    all_ = gpu["all"]
    errs = {k: LP.rel(sum(gpu[s][k] for s in LP.LOSSES), v) for k, v in all_.items()
            if not LP.is_shift_invariant(k) and float(v.abs().max()) > 0}
    record(f"{case}/sum", dict(LP.summary(errs), bar=LP.SUM_BAR))
    worst = max(errs.items(), key=lambda kv: kv[1])
    assert worst[1] <= LP.SUM_BAR, worst


@pytest.mark.parametrize("subset", ["ctr", "all"])
def test_side_stream_matches_one_stream(subset, tiny_cfg, monkeypatch):
    """The language-only backward runs on a side stream, concurrently with the joint backward, and both accumulate into
    encoder/.  With MERLOT_NO_SIDE_STREAM=1 everything runs on one stream: the gradients may differ only as two default runs
    do (the order of fp32 atomic adds).  Bar: loss_paths_oracle.SIDE_BAR, from the repeat spread measured on the H100, with a
    floor of 1e-6 relative."""
    r, gpu, _ = _results("eval", tiny_cfg)
    a, b = gpu[subset], r.grads(subset)
    monkeypatch.setenv("MERLOT_NO_SIDE_STREAM", "1")
    one = r.grads(subset)
    keys = [k for k, v in a.items() if float(v.abs().max()) > 0 and not LP.is_shift_invariant(k)]
    rep = {k: LP.rel(b[k], a[k]) for k in keys}
    one_s = {k: LP.rel(one[k], a[k]) for k in keys}
    record(f"side_stream/{subset}", {"repeat": LP.summary(rep), "one_stream": LP.summary(one_s), "bar": LP.SIDE_BAR})
    assert max(rep.values()) <= LP.SIDE_BAR, LP.summary(rep)
    assert max(one_s.values()) <= LP.SIDE_BAR, LP.summary(one_s)
