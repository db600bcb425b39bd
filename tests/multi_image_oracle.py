"""TEST INFRASTRUCTURE ONLY.  The reference's several-images-per-text input restated on the CPU: `num_imgs` and `img_mask` of
MerlotModel (model/modeling.py:64,84,106-122,152-158,186-203) and vision_pos_emb's unshuffled branch (:299-315,336), over the
primitives of oracle/merlot_oracle.py (vision_transformer_backbone, layer_norm, position_embedder2d, transformer and
MerlotOracle.embed_words, which it calls unchanged).

This is the joint-encoder forward that a downstream head builds on: no mask_input, no shuffled_idx_img (the reference asserts
num_imgs == 1 there, :319), no disable_pairwise_lang_attn.  With num_imgs = 1 and img_mask = None it is MerlotOracle's
forward with mask_input=False (tests/test_multi_image_host.py checks that they agree bit for bit).

All `file:line` citations are relative to the reference repository (rowanz/merlot)."""
from __future__ import annotations

import copy

import torch

from oracle import merlot_oracle as O


def image_pos_emb(p, ncg_ni: int, vcl: int, num_h: int, num_w: int) -> torch.Tensor:
    """vision_pos_emb(shuffled_idx_img=None) (:299-337) for ncg_ni = num_chunks_in_group * num_imgs images: [1, ncg_ni * vcl, H].
    Token t of image i gets img_idx_pe[i] + final_pe[t] (final_pe = the 2-D table with one cls row first)."""
    table = p["vision_backbone/img_idx_pe"]
    my_pe = table[:ncg_ni]  # position_embedder(num_chunks_in_group * num_imgs) (:305-311): rows 0 .. ncg_ni - 1
    my_pe = my_pe[:, None].expand(ncg_ni, vcl, -1).reshape(1, ncg_ni * vcl, -1)  # tile over the image's tokens (:314-315)
    pe2d = O.position_embedder2d(p, "vision_backbone/final_pe", num_h, num_w, 1)  # :327-335
    return my_pe + pe2d.repeat(ncg_ni, 1)[None]  # :336


class MultiImageOracle:
    """image: [N, h, w, 3] float in [0, 1]; input_ids: int [batch, Lc] or [batch, num_chunks, Lc]; img_mask: None or any bool /
    integer tensor of B // num_texts * num_imgs entries (non-zero = valid).  dropout: None (eval) or the hook of
    oracle/dropout_mask.py (keys as MerlotOracle's).  Exposes encoder_info, encoder_hidden_states, encoder_pieces,
    attention_log, is_valid [B, P * num_imgs + L] and the shape properties."""

    def __init__(self, config: dict, params, image, input_ids, img_mask=None, log_attention_probs=True, dropout=None):
        self.config = cfg = copy.deepcopy(config)
        self.p = params
        self.hidden_size, self.vocab_size = cfg["hidden_size"], cfg["vocab_size"]
        if input_ids.dim() == 2:  # :72-77
            self.num_chunks = self.num_chunks_in_group = 1
            self.batch_size, self.lang_chunk_length = input_ids.shape
            self.input_ids = input_ids[:, None]
        else:
            self.input_ids = input_ids
            self.batch_size, self.num_chunks, self.lang_chunk_length = input_ids.shape
            self.num_chunks_in_group = cfg.get("num_chunks_in_group", self.num_chunks)
            assert self.num_chunks % self.num_chunks_in_group == 0  # :82
        self.num_imgs = ni = cfg.get("num_imgs", 1)  # :84
        self.num_texts = nt = cfg.get("num_texts", 1)  # :85
        self.img_batch_size = self.batch_size // nt  # :86
        H, B, dt = self.hidden_size, self.B, image.dtype

        vit = self.vision_transformer_info = O.vision_transformer_backbone(image, cfg, params, dropout)  # :96
        self.img_trg_h = vit["cls"][:, 1]  # :99
        feats = torch.cat([vit["cls"][:, 0, None], vit["seq"]], 1)  # :101-104
        self.viz_chunk_length = vit["num_h"] * vit["num_w"] + 1
        if img_mask is None:  # :106-107
            img_mask = torch.ones(B // nt, ni, dtype=torch.bool)
        else:  # :108-109
            img_mask = img_mask.reshape(B // nt, ni) != 0
        if ni > 1 or nt > 1:  # :111-119
            feats = feats.reshape(self.img_batch_size, ni, *feats.shape[1:])  # :112
            if nt > 1:
                feats = feats[:, None].expand(-1, nt, *feats.shape[1:]).reshape(B, *feats.shape[1:])  # :116-117
                img_mask = img_mask[:, None].expand(-1, nt, -1).reshape(B, ni)  # :118-119
        feats = feats.reshape(B, self.P * ni, H)  # :121
        viz_valid = img_mask[:, :, None].expand(B, ni, self.P).reshape(B, self.P * ni)  # :122
        feats = feats + image_pos_emb(params, self.num_chunks_in_group * ni, self.viz_chunk_length, vit["num_h"], vit["num_w"])  # :125
        feats = O.layer_norm(feats, params, "vision_backbone/LayerNorm_final_ln")  # :126
        pieces = [{"name": "viz", "x": feats, "is_valid": viz_valid}]  # :129-133

        ids = self.input_ids.reshape(B, self.L)  # :141-143
        pieces.append({"name": "lang", "x": O.MerlotOracle.embed_words(self, ids, dropout=dropout), "is_valid": ids != 0})  # :145-149
        enc_in = torch.cat([x["x"] for x in pieces], 1)  # :151
        self.is_valid = is_valid = torch.cat([x["is_valid"] for x in pieces], 1)  # :152
        attn_mask = (is_valid[:, None] & is_valid[:, :, None]).to(dt)  # :158,170
        self.encoder_info = O.transformer(enc_in, attn_mask, params, "encoder", cfg["num_hidden_layers"], cfg["num_attention_heads"],
                                          return_attn_probs=log_attention_probs, dropout=O._scoped(dropout, "joint"))  # :171-174
        self.encoder_hidden_states = {}
        cur = 0
        for x in pieces:  # :176-184
            x["start"], x["end"] = cur, cur + x["x"].shape[1]
            cur = x["end"]
            self.encoder_hidden_states[x["name"]] = self.encoder_info["hidden_state"][:, x["start"]:x["end"]]
        self.encoder_pieces = pieces
        if log_attention_probs:  # :186-203
            sap = self.encoder_info["self_attn_probs"].mean(1)
            vf = is_valid.to(dt)
            sap = sap * (vf[:, None] * vf[:, :, None])
            sap = sap.mean(0)
            sap = sap / sap.sum()
            attns = {}
            for x_to in pieces:
                for x_from in pieces:
                    attns[f"{x_from['name']}2{x_to['name']}"] = sap[x_to["start"]:x_to["end"], x_from["start"]:x_from["end"]].sum()
            self.attention_log = {f"encoder/{k}": v for k, v in sorted(attns.items())}

    # shapes (:234-248)
    @property
    def B(self):
        return self.batch_size * (self.num_chunks // self.num_chunks_in_group)

    @property
    def L(self):
        return self.lang_chunk_length * self.num_chunks_in_group

    @property
    def P(self):
        return self.viz_chunk_length * self.num_chunks_in_group
