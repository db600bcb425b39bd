"""Host checks behind tests/test_gpu_trajectory.py (no GPU): AdamOracle continued from a saved state is the uninterrupted
oracle, the chosen schedule crosses the warm-up boundary with distinct learning rates, and the wrong-reference seeds are
not the step's own."""
import numpy as np
import pytest
import torch

from merlot_b200.config import replica_seed
from merlot_b200.optimization import learning_rate_scale
from oracle import merlot_oracle as O
from tests import test_gpu_trajectory as TJ


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


@pytest.mark.parametrize("use_bf16", [True, False])
@pytest.mark.parametrize("j", [0, 1, 3])
def test_adam_oracle_from_state_continues_the_run(use_bf16, j):
    """k steps in one run against j steps, a restart from (p, m, v, global_step) and k - j more: the same bits.  The run
    crosses the warm-up boundary, decays the learning rate and decays the weights of one tensor."""
    cfg = dict(TJ.OCFG, use_bfloat16_adam=use_bf16, param_overrides=[[["bias"], {"weight_decay_rate": 0}]])
    g = torch.Generator().manual_seed(4)
    p0 = {"w/kernel": torch.randn(257, 3, generator=g) * 0.02, "w/bias": torch.randn(129, generator=g) * 0.02}
    K = TJ.TRAIN_STEPS - 1
    grads = [{k: torch.randn(v.shape, generator=g) * 10.0 ** float(torch.randint(-6, 1, (1,), generator=g)) for k, v in p0.items()}
             for _ in range(K)]
    whole_p = {k: v.clone() for k, v in p0.items()}
    whole = O.AdamOracle(whole_p, cfg)
    for gr in grads:
        whole.apply_gradients(whole_p, gr)
    part_p = {k: v.clone() for k, v in p0.items()}
    part = O.AdamOracle(part_p, cfg)
    for gr in grads[:j]:
        part.apply_gradients(part_p, gr)
    rest_p = {k: v.clone() for k, v in part_p.items()}
    rest = O.AdamOracle.from_state(rest_p, cfg, part.m, part.v, part.global_step)
    assert rest.global_step == j and all(rest.m[k] is not part.m[k] for k in p0)  # a copy, not the same tensors
    for gr in grads[j:]:
        rest.apply_gradients(rest_p, gr)
    assert rest.global_step == whole.global_step == K
    for k in p0:
        assert rest.m[k].dtype == (torch.bfloat16 if use_bf16 else torch.float32)
        assert torch.equal(_bits(rest_p[k]), _bits(whole_p[k])), k
        assert torch.equal(_bits(rest.m[k]), _bits(whole.m[k])), k
        assert torch.equal(_bits(rest.v[k]), _bits(whole.v[k])), k
    assert not torch.equal(whole_p["w/kernel"], p0["w/kernel"])


def test_adam_oracle_from_state_refuses_other_storage():
    cfg = dict(TJ.OCFG, use_bfloat16_adam=True)
    p = {"w/kernel": torch.zeros(4, 2)}
    m32 = {"w/kernel": torch.zeros(4, 2)}
    with pytest.raises(ValueError, match="w/kernel"):
        O.AdamOracle.from_state(p, cfg, m32, m32, 3)
    with pytest.raises(ValueError, match="w/kernel"):
        O.AdamOracle.from_state(p, dict(cfg, use_bfloat16_adam=False), {"w/kernel": torch.zeros(8)}, {"w/kernel": torch.zeros(8)}, 3)


@pytest.mark.parametrize("name", list(TJ.VARIANTS))
def test_schedule_crosses_the_warmup_boundary(name):
    """Pretraining variants: scale 0 at step 0 (the warm-up), then distinct non-zero scales, both sides of the boundary.
    VCR (warm-up 0): distinct non-zero scales from step 0.  The test's scales are the product's learning_rate_scale."""
    c = TJ.optimizer_cfg(name)
    s = TJ.lr_scales(name)
    assert s == [float(learning_rate_scale(k, c["num_train_steps"], c["num_warmup_steps"])) for k in range(len(s))]
    assert len(set(s)) == len(s) and len(s) == TJ.VARIANTS[name]["steps"]
    if name == "vcr":
        assert c["num_warmup_steps"] == 0 and min(s) > 0
        return
    W = c["num_warmup_steps"]
    assert s[0] == 0.0 and min(s[1:]) > 0
    assert 0 < W < len(s) and s[W - 1] < s[W]  # step W, the first after the warm-up, is in the run
    assert all(a > b for a, b in zip(s[W:], s[W + 1:]))  # and the decay follows it
    assert len(s) < c["num_train_steps"]  # every step is before the end of the decay


@pytest.mark.parametrize("name", list(TJ.VARIANTS))
def test_wrong_reference_seeds_are_not_the_steps_own(name):
    """The test's seeds are config.replica_seed's on one GPU (A = 2 in the clipped accumulation), and the previous step's
    seeds, which the seed-not-advanced reference uses, share no seed with the step's own."""
    A = TJ.VARIANTS[name].get("accum", 1)
    seen = set()
    for k in range(TJ.VARIANTS[name]["steps"]):
        mine = TJ.step_seeds(name, k)
        assert mine == [replica_seed(TJ.SEED, k, 1, A, 0, j) for j in range(A)]
        assert not seen & set(mine)
        if k > 0:
            assert not set(TJ.step_seeds(name, k - 1)) & set(mine)
        seen |= set(mine)
    assert TJ.SEED >> 32  # the seed's high word reaches the kernels


def test_learning_rate_metric_rounding():
    """metrics['learning_rate'] is float32(lr) * float32 scale in float32 (AdamOptimizer.current_lr); the test's expectation
    rounds the same way and is not the double product."""
    k = 1
    want = float(np.float32(np.float32(TJ.LR) * O.lr_scale(k, TJ.TRAIN_STEPS, TJ.WARMUP)))
    assert want == float(np.float32(want)) and want > 0
