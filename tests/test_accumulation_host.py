"""Gradient accumulation on the host (no GPU): the micro-batch count from the configuration, the virtual replicas' seeds,
the rank-level contrastive head (labels and coefficients over A micro-batches) against the replica oracle, and the trainer
drawing A batches per optimizer step."""
import pytest
import torch

from merlot_b200.config import micro_batching, replica_seed


def test_micro_batching_without_the_key_is_one_batch_per_rank():
    assert micro_batching({"train_batch_size": 1024}, 8) == (1, 128)
    assert micro_batching({}, 1) == (1, 8)
    assert micro_batching({}, 1, default_batch_size=64) == (1, 64)
    assert micro_batching({"train_batch_size": 4}, 8) == (1, 1)  # as before: at least one example per rank


@pytest.mark.parametrize("tbs,world,m,A", [(1024, 8, 16, 8), (1024, 8, 128, 1), (64, 1, 8, 8), (6, 1, 2, 3), (12, 2, 3, 2)])
def test_micro_batching_accumulation_steps(tbs, world, m, A):
    assert micro_batching({"train_batch_size": tbs, "micro_batch_size": m}, world) == (A, m)


@pytest.mark.parametrize("tbs,world,m", [(1000, 8, 16), (1024, 8, 256), (8, 8, 2), (6, 4, 1), (64, 1, 0), (64, 1, -8)])
def test_micro_batching_rejects_a_batch_that_does_not_split(tbs, world, m):
    with pytest.raises(ValueError) as e:
        micro_batching({"train_batch_size": tbs, "micro_batch_size": m}, world)
    msg = str(e.value)
    assert f"train_batch_size {tbs}" in msg and f"world {world}" in msg and f"micro_batch_size {m}" in msg


def test_replica_seed_with_one_micro_batch_is_the_data_parallel_seed():
    for seed in (0, 7):
        for step in range(5):
            for world in (1, 2, 8):
                for rank in range(world):
                    assert replica_seed(seed, step, world, 1, rank, 0) == seed + step * world + rank


def test_replica_seeds_are_distinct_and_consecutive():
    world, A = 3, 4
    for step in range(4):
        got = sorted(replica_seed(5, step, world, A, r, j) for r in range(world) for j in range(A))
        assert got == list(range(5 + step * world * A, 5 + (step + 1) * world * A))
    # virtual replica v = rank * A + j
    assert replica_seed(0, 0, world, A, 2, 1) == 2 * A + 1


# ---- the rank-level contrastive head on the CPU: host logic of modeling.contrastive_head with CPU stand-ins for its kernels
class _CpuOps:
    """CPU stand-ins for the kernels of the contrastive head, in float64; K16's operand layouts are followed exactly, so the
    head's K concatenations and strides are what is checked."""

    @staticmethod
    def _split(v):
        h = v.to(torch.bfloat16)
        return h, (v - h.float()).to(torch.bfloat16)

    @staticmethod
    def ctr_split(x, out, ld, seg_stride, lo_mask):
        rows, C = x.shape
        h, l = _CpuOps._split(x)
        flat = out.view(-1)
        for s in range(3):
            seg = torch.as_strided(flat, (rows, C), (ld, 1), s * seg_stride)
            seg.copy_(l if (lo_mask >> s) & 1 else h)

    @staticmethod
    def gemm(a, b, *, a_mn_major=False, b_mn_major=False, out=None, alpha=1.0, M=None, N=None, K=None, **kw):
        A = (a[:K, :M].t() if a_mn_major else a[:M, :K]).double()
        B = (b[:K, :N] if b_mn_major else b[:N, :K].t()).double()
        out[:M, :N] = (alpha * A @ B).float()

    @staticmethod
    def ctr_dlogits(logits, labels, C, lse, coeff, scale, dsh, dsv):
        n = logits.shape[0]
        p = torch.softmax(logits[:, :C].double(), 1)
        p[torch.arange(n), labels.long()] -= 1.0
        h, l = _CpuOps._split((p * coeff.double()[:, None] * scale).float())
        dsh[:, :C], dsh[:, C:2 * C], dsh[:, 2 * C:3 * C] = h, h, l
        dsv[:n, :C], dsv[n:2 * n, :C], dsv[2 * n:3 * n, :C] = h, h, l

    @staticmethod
    def softmax_ce_fwd(logits, labels, Cn, loss, lse, correct=None):
        z = logits[:, :Cn].double()
        lse[:] = torch.logsumexp(z, 1).float()
        loss[:] = (torch.logsumexp(z, 1) - z.gather(1, labels.long()[:, None])[:, 0]).float()

    @staticmethod
    def weighted_loss(per_row, correct, weights, nz_labels, denom_mode, scale, out2, coeff):
        assert weights is None and nz_labels is None and denom_mode == 0
        R = per_row.numel()
        out2[0] = per_row.double().sum() / R
        coeff[:] = scale / R

    @staticmethod
    def axpby(x, y, a=1.0, b=1.0):
        y.view(-1)[:] = a * x.reshape(-1) + (b * y.reshape(-1) if b else 0.0)


class _Store:
    device = "cpu"


def _features(replicas, n, Cs, seed):
    g = torch.Generator().manual_seed(seed)
    f = torch.nn.functional.normalize(torch.randn(replicas * n, Cs, generator=g), dim=1)
    return f


def _oracle_replicas(lang, viz, n, cfg):
    """Per-replica contrastive losses of oracle.contrastive_loss_replicas over replicas holding rows v*n..(v+1)*n."""
    from oracle import merlot_oracle as O

    class R:
        def __init__(self, v):
            self.config = cfg
            self._ctr_feats = (lang[v * n:(v + 1) * n], viz[v * n:(v + 1) * n])

    models = [R(v) for v in range(lang.shape[0] // n)]
    return [O.contrastive_loss_replicas(models, v)[0] for v in range(len(models))]


@pytest.mark.parametrize("world,A,n", [(1, 1, 4), (1, 3, 4), (2, 2, 3), (3, 2, 2)])
def test_contrastive_head_over_micro_batches_is_the_replica_oracle(monkeypatch, world, A, n):
    from merlot_b200 import modeling as M
    monkeypatch.setattr(M, "ops", _CpuOps)
    cfg = {"contrast_temp": 0.07, "contrast_coef": 0.5}
    Cs = 8
    lang_all, viz_all = _features(world * A, n, Cs, 1), _features(world * A, n, Cs, 2)
    lang_leaf, viz_leaf = lang_all.double().requires_grad_(True), viz_all.double().requires_grad_(True)
    per = _oracle_replicas(lang_leaf, viz_leaf, n, cfg)
    sum(per).backward()  # the accumulated gradient: every replica's loss, unscaled (AdamW applies 1 / (world * A))
    rows = A * n
    d_local, d_cols = [], []
    for rank in range(world):
        mine = slice(rank * rows, (rank + 1) * rows)
        lang_mine, viz_mine = lang_all[mine].contiguous(), viz_all[mine].contiguous()

        class Dist:
            """Every rank's rows are known here: the all-gather is the full feature matrix.  The reduce-scatter records this
            rank's gradient of all columns and contributes nothing; the test sums the records over ranks below."""

            def all_gather_rows(self, x):
                return (lang_all if x is lang_mine else viz_all).clone()

            def reduce_scatter_rows(self, x_all):
                cols.append(x_all.clone())
                return torch.zeros(rows, x_all.shape[1])

        d, cols = Dist(), []
        d.world, d.rank = world, rank
        dist = d if world > 1 else None
        bufs = M._Buffers(_Store())
        info, outs = M.contrastive_head(bufs, cfg, dist, lang_mine, viz_mine, n)
        # labels: virtual replica v = rank * A + j labels its row i with v * n + i
        assert info["labels"].tolist() == list(range(rank * rows, (rank + 1) * rows))
        # reported: the mean over this rank's replicas
        mean_mine = sum(float(per[rank * A + j].detach()) for j in range(A)) / A
        assert abs(float(outs["loss_all"]) - mean_mine) <= 1e-5 * abs(mean_mine)
        d_feat = M.contrastive_head_bwd(bufs, dist, info)
        d_local.append({k: v.clone() for k, v in d_feat.items()})
        d_cols.append(dict(zip(("lang", "viz"), cols)))
    # each rank's rows: its own rows' gradient plus the sum over ranks of the gradient of its columns (the reduce-scatter)
    for rank in range(world):
        mine = slice(rank * rows, (rank + 1) * rows)
        for k, leaf in (("lang", lang_leaf), ("viz", viz_leaf)):
            got = d_local[rank][k] + (sum(c[k][mine] for c in d_cols) if world > 1 else 0.0)
            ref = leaf.grad[mine].float()
            assert (got - ref).norm() <= 1e-5 * ref.norm(), (rank, k)


def test_contrastive_head_rejects_a_partial_replica(monkeypatch):
    from merlot_b200 import modeling as M
    monkeypatch.setattr(M, "ops", _CpuOps)
    f = _features(1, 5, 8, 0)
    with pytest.raises(ValueError, match="whole number of replicas"):
        M.contrastive_head(M._Buffers(_Store()), {}, None, f, f, 2)


# ---- the trainer draws A micro-batches per optimizer step
class _FakeStore:
    task = "vcr"
    entries = {}

    def __init__(self):
        self.global_step = 0

    def save_checkpoint(self, prefix, skip=()):
        pass


def _run_main(tmp_path, monkeypatch, device, steps=2, pipeline=False):
    import yaml
    from merlot_b200 import train, vcr_input
    calls, draws = [], []

    def builder(config, dist=None):
        store = _FakeStore()

        def model_fn(features, labels=None, mode="train", params=None):
            calls.append(features)

            def train_op():
                store.global_step += 1
            return train.StepSpec(None, [torch.zeros(())], {"learning_rate": 0.0}, train_op)
        model_fn.store = store
        return model_fn

    def make_batch(config, batch_size, seed=0):
        draws.append((batch_size, seed))
        return {"n": batch_size, "seed": seed}

    class Pipe:
        def __init__(self, batch_size):
            self.batch_size, self.k = batch_size, 0

        def __next__(self):
            self.k += 1
            return {"n": self.batch_size, "k": self.k}

        def close(self):
            pass

    monkeypatch.setattr(train, "_step_for", lambda config: (builder, make_batch))
    if pipeline:
        monkeypatch.setattr(train, "train_files", lambda data: ["x"])
        monkeypatch.setattr(vcr_input, "input_fn_builder", lambda config, batch_size=None, **kw: Pipe(batch_size))
    cfg = {"data": {}, "model": {}, "optimizer": {"num_train_steps": steps}, "device": dict(device, output_dir=str(tmp_path / "o"))}
    path = tmp_path / "c.yaml"
    path.write_text(yaml.safe_dump(cfg))
    train.main([str(path)])
    return calls, draws


def test_trainer_without_micro_batch_size_draws_one_batch(tmp_path, monkeypatch):
    calls, draws = _run_main(tmp_path, monkeypatch, {"train_batch_size": 6})
    assert calls == [{"n": 6, "seed": 0}, {"n": 6, "seed": 1}]  # one dict per step, as before


def test_trainer_draws_A_micro_batches_per_step(tmp_path, monkeypatch):
    calls, draws = _run_main(tmp_path, monkeypatch, {"train_batch_size": 6, "micro_batch_size": 2}, steps=2)
    assert len(calls) == 2 and all(isinstance(c, list) and len(c) == 3 for c in calls)
    assert all(f["n"] == 2 for c in calls for f in c)
    seeds = [f["seed"] for c in calls for f in c]
    assert seeds == list(range(6))  # every micro-batch of every step is a different batch


def test_trainer_pipeline_is_built_at_the_micro_batch(tmp_path, monkeypatch):
    calls, _ = _run_main(tmp_path, monkeypatch, {"train_batch_size": 8, "micro_batch_size": 4}, steps=2, pipeline=True)
    assert [[f["k"] for f in c] for c in calls] == [[1, 2], [3, 4]]
    assert all(f["n"] == 4 for c in calls for f in c)


def test_trainer_rejects_a_batch_that_does_not_split(tmp_path, monkeypatch):
    with pytest.raises(ValueError, match="train_batch_size 6 is not world 1 x A x micro_batch_size 4"):
        _run_main(tmp_path, monkeypatch, {"train_batch_size": 6, "micro_batch_size": 4})


def test_input_builders_default_to_the_micro_batch(tmp_path, monkeypatch):
    from merlot_b200 import dataloader as D
    from merlot_b200 import vcr_input as VI
    from merlot_b200.config import NeatConfig
    seen = {}
    monkeypatch.setattr(D, "InputPipeline", lambda config, files, batch_size, **kw: seen.setdefault("pre", batch_size))
    monkeypatch.setattr(VI, "VCRTrainPipeline", lambda config, files, batch_size, **kw: seen.setdefault("vcr", batch_size))
    for name in ("a", "b"):  # one file per rank
        (tmp_path / f"{name}.tfrecord").write_bytes(b"")
    cfg = NeatConfig.from_dict({"data": {"train_file": str(tmp_path / "*.tfrecord")}, "model": {}, "optimizer": {},
                                "device": {"output_dir": "/tmp/unused", "train_batch_size": 16, "micro_batch_size": 4}})
    D.input_fn_builder(cfg, True, rank=0, world=2)
    VI.input_fn_builder(cfg, True, rank=0, world=2)
    assert seen == {"pre": 4, "vcr": 4}
