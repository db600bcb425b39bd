"""The oracle's reading of `share_params: False` (model/modeling.py:171-172, 356-379): `langonly_reps` runs its own stack,
`langonly_encoder/` of num_lang_transformer_hidden_layers layers, and the joint `encoder/` has num_hidden_layers.

`param_shapes` and `langonly_reps` extend oracle.merlot_oracle's functions of the same names; with share_params True (or
the key absent) they return exactly what those return.  `use_separate_oracle(monkeypatch)` puts them into that module for
one test, so every helper written against it (init_params, MerlotOracle, pretrain_losses, the step-parity helpers of the
GPU tests) runs the separate encoder unchanged."""
from __future__ import annotations

from oracle import merlot_oracle as O

_shared_param_shapes = O.param_shapes
_shared_langonly_reps = O.MerlotOracle.langonly_reps


def param_shapes(cfg: dict):
    """O.param_shapes, with a `langonly_encoder/` stack right after `encoder/` when share_params is False."""
    if cfg.get("share_params", True):
        return _shared_param_shapes(cfg)
    joint = _shared_param_shapes(dict(cfg, num_lang_transformer_hidden_layers=0))  # encoder/: num_hidden_layers layers
    lo = _shared_param_shapes(dict(cfg, num_hidden_layers=cfg["num_lang_transformer_hidden_layers"],
                                   num_lang_transformer_hidden_layers=0))
    lo = {"langonly_encoder/" + k[len("encoder/"):]: v for k, v in lo.items() if k.startswith("encoder/")}
    out = {}
    for k, v in joint.items():
        out[k] = v
        if k == "encoder/LayerNorm_ln_final/beta":
            out.update(lo)
    return out


def langonly_reps(self, dropout=None):
    """MerlotOracle.langonly_reps (:339-379) on the `langonly_encoder` scope when share_params is False."""
    cfg = self.config
    if cfg.get("share_params", True):
        return _shared_langonly_reps(self, dropout)
    g = cfg.get("langonly_num_chunks_in_group", self.num_chunks)
    assert self.num_chunks // g > 0 and self.num_chunks % g == 0
    ids = self.input_ids.reshape(self.batch_size * (self.num_chunks // g), self.lang_chunk_length * g)
    emb = self.embed_words(ids, "langonly_embeddings", dropout)
    valid = ids != 0
    mask = (valid[:, None] & valid[:, :, None]).to(emb.dtype)
    info = O.transformer(emb, mask, self.p, "langonly_encoder", cfg["num_lang_transformer_hidden_layers"],
                         cfg["num_attention_heads"], return_attn_probs=True, dropout=O._scoped(dropout, "langonly"))
    pool = info["_hidden_state_flat"].reshape(self.batch_size * self.num_chunks, self.lang_chunk_length, -1)[:, 0]
    return pool, info


def use_separate_oracle(monkeypatch):
    monkeypatch.setattr(O, "param_shapes", param_shapes)
    monkeypatch.setattr(O.MerlotOracle, "langonly_reps", langonly_reps)
