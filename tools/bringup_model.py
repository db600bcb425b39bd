"""GPU bring-up of the whole MerlotModel path against the oracle on a tiny config (test infrastructure).
Prints per-tensor errors for forward activations, losses and every parameter gradient."""
import sys
import time

import torch

sys.path.insert(0, ".")
from merlot_b200.modeling import MerlotModel  # noqa: E402
from merlot_b200.params import ParamStore  # noqa: E402
from oracle import merlot_oracle as O  # noqa: E402


def tiny_cfg(**over):
    cfg = dict(use_bfloat16=True, hidden_size=128, vocab_size=1000, patch_size=16, spatial_pool_size=2, num_attention_heads=2,
               num_hidden_layers=2, num_vision_transformer_hidden_layers=2, num_lang_transformer_hidden_layers=2,
               intermediate_size=256, initializer_range=0.02, hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.0,
               max_position_embeddings=64, num_chunks_in_group=2, do_projection=True, do_bias=True, contrastive_size=128,
               contrast_coef=0.25, contrast_temp=0.05, image_shuffle_prob=0.4, masking_rate=0.2, resnet_layers=[])
    cfg.update(over)
    return cfg


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def synth(cfg, batch, num_chunks, Lc, h0, w0, seed):
    g = torch.Generator().manual_seed(seed)
    image = torch.rand(batch * num_chunks, h0, w0, 3, generator=g).bfloat16().float()
    ids = torch.randint(100, cfg["vocab_size"], (batch, num_chunks, Lc), generator=g)
    ids[:, :, 0] = O.START
    lens = torch.randint(Lc // 2, Lc + 1, (batch, num_chunks), generator=g)
    ids = ids * (torch.arange(Lc)[None, None] < lens[..., None])
    ncg = cfg["num_chunks_in_group"]
    B = batch * num_chunks // ncg
    shuf = torch.arange(ncg).repeat(B)
    shuf[:ncg] = 16 + torch.randperm(ncg, generator=g)
    shuf[ncg:2 * ncg] = 64 + torch.randperm(ncg, generator=g)
    vid = torch.zeros(B, ncg, dtype=torch.int64)
    vid[0, ncg // 2:] = 1
    return image, ids.int(), shuf.int(), vid.int()


def main():
    dev = "cuda"
    cfg = tiny_cfg()
    batch, num_chunks, Lc, h0, w0 = 2, 4, 16, 64, 96
    image, ids, shuf, vid = synth(cfg, batch, num_chunks, Lc, h0, w0, 0)
    params = O.init_params(cfg, seed=1, perturb=0.05)
    # the bf16 compute copy is what the GPU multiplies with: give the oracle the same rounded matrices
    params_r = {k: (v.bfloat16().float() if (k.endswith("kernel") or k == "word_embeddings/word_embeddings") else v)
                for k, v in params.items()}
    store = ParamStore(cfg, device=dev)
    store.load_tf_dict(params_r)

    B = batch * num_chunks // cfg["num_chunks_in_group"]
    Lj = Lc * cfg["num_chunks_in_group"]
    draws = O.make_mask_draws(B, Lj, int(Lj * 0.2), cfg["vocab_size"], seed=5)
    ok = True

    # ---------------- forward, eval mode (dropout 0), with masking ----------------
    t0 = time.time()
    m = MerlotModel(cfg, is_training=False, use_tpu=False, image=image.to(dev), input_ids=ids.to(dev), mask_input=True,
                    shuffled_idx_img=shuf.to(dev), params=store, mask_draws=draws, save_for_backward=True)
    torch.cuda.synchronize()
    print(f"gpu forward {time.time() - t0:.2f}s", flush=True)
    leaf = {k: v.clone().requires_grad_(True) for k, v in params_r.items()}
    om = O.MerlotOracle(cfg, leaf, image, ids, mask_input=True, shuffled_idx_img=shuf, mask_draws=draws)
    e = rel(m.lang_transformer_info["attention_summs"], om.attention_summs)
    print(f"attention_summs rel={e:.3e}")
    same_ids = torch.equal(m.lang_mask_info["masked_ids"].cpu().reshape(B, Lj), om.lang_mask_info["masked_ids"])
    same_idx = torch.equal(m.lang_mask_info["masked_idx"].cpu(), om.lang_mask_info["masked_idx"])
    print(f"mask from GPU attention sums identical to oracle's: ids={same_ids} idx={same_idx}")
    # masking kernel bit-exactness given the ORACLE's attention sums
    from merlot_b200 import ops
    m2_ids = torch.empty(B, Lj, dtype=torch.int32, device=dev)
    m2_idx = torch.empty(B, int(Lj * 0.2), dtype=torch.int32, device=dev)
    mi = O.mask_inputs(ids.reshape(B, Lj), om.attention_summs.detach(), cfg, draws)
    import numpy as np
    w = torch.tensor([1.0, 0.0]) * np.float32(mi["topk_val"] - 0.01) + np.float32(0.01)
    consts = (float(np.float32(mi["topk_val"] - 0.01)), float(np.float32(0.01)), float(torch.log(w)[0]), float(torch.log(w)[1]), float(w.max()))
    ops.mask_inputs(ids.reshape(B, Lj).to(dev), om.attention_summs.detach().float().contiguous().to(dev),
                    {k: v.to(dev) for k, v in draws.items()}, m2_ids, m2_idx, None, int(Lj * 0.2), int(Lj * 0.2), True, 1, consts)
    bit = torch.equal(m2_ids.cpu(), mi["masked_ids"]) and torch.equal(m2_idx.cpu(), mi["masked_idx"])
    print(f"{'OK  ' if bit else 'FAIL'} mask_inputs kernel bit-exact given oracle attention sums: {bit}")
    ok &= bit
    if not (same_ids and same_idx):  # feed the GPU's mask to the oracle so the rest is comparable
        om = O.MerlotOracle(cfg, leaf, image, ids, mask_input=True, shuffled_idx_img=shuf,
                            mask_override={"masked_ids": m.lang_mask_info["masked_ids"].cpu().reshape(B, Lj),
                                           "masked_idx": m.lang_mask_info["masked_idx"].cpu()})
    for name in ("viz", "lang"):
        e = rel(m.encoder_hidden_states[name], om.encoder_hidden_states[name])
        print(f"{'OK  ' if e < 2e-2 else 'FAIL'} encoder_hidden_states[{name}] rel={e:.3e}")
        ok &= e < 2e-2
    e1, e2 = rel(m.img_trg_h, om.img_trg_h), rel(m.lang_trg_h, om.lang_trg_h)
    print(f"img_trg_h rel={e1:.3e} lang_trg_h rel={e2:.3e}")

    # ---------------- losses ----------------
    ll, linfo = m.mask_loss()
    cl, cinfo = m.contrastive_loss()
    tl, tinfo = m.temporal_loss(shuf.to(dev), vid.to(dev))
    torch.cuda.synchronize()
    o_total, oinfo = O.pretrain_losses(om, shuf, vid)
    pairs = [("lang/loss", ll, oinfo["lang"]["loss"]), ("lang/acc", linfo["acc"], oinfo["lang"]["acc"]),
             ("contr/lang_to_viz", cinfo["lang_to_viz"], oinfo["contr"]["lang_to_viz"]),
             ("contr/viz_to_lang", cinfo["viz_to_lang"], oinfo["contr"]["viz_to_lang"]),
             ("contr/loss_all", cl, oinfo["contr"]["loss_all"]),
             ("temporal/lang_viz_loss", tinfo["lang_viz_loss"], oinfo["temporal"]["lang_viz_loss"]),
             ("temporal/viz_viz_loss", tinfo["viz_viz_loss"], oinfo["temporal"]["viz_viz_loss"]),
             ("temporal/lang_viz_acc", tinfo["lang_viz_acc"], oinfo["temporal"]["lang_viz_acc"]),
             ("temporal/loss", tl, oinfo["temporal"]["loss"])]
    for name, a, b in pairs:
        a, b = float(a), float(b)
        r = abs(a - b) / (abs(b) + 1e-12)
        good = r < 5e-3 or "acc" in name
        print(f"{'OK  ' if good else 'FAIL'} {name}: gpu={a:.6f} oracle={b:.6f} rel={r:.2e}")
        ok &= good
    total_gpu = float(ll) + float(cl) + float(tl)
    print(f"total loss gpu={total_gpu:.6f} oracle={float(o_total):.6f} rel={abs(total_gpu - float(o_total)) / abs(float(o_total)):.2e}")

    # ---------------- backward ----------------
    store.g.zero_()
    m.backward()
    torch.cuda.synchronize()
    o_total.backward()
    grads = store.to_tf_dict("g")
    worst = []
    for k in sorted(leaf):
        g_or = leaf[k].grad
        if g_or is None:
            continue
        r = rel(grads[k], g_or)
        worst.append((r, k, float(g_or.norm())))
    worst.sort(reverse=True)
    nbad = sum(1 for r, k, n in worst if r > 5e-2 and n > 1e-7)
    print(f"gradients: {len(worst)} tensors, {nbad} with rel>5e-2; worst 25:")
    for r, k, n in worst[:25]:
        print(f"   {r:.3e}  |g|={n:.3e}  {k}")
    print("best 5:")
    for r, k, n in worst[-5:]:
        print(f"   {r:.3e}  |g|={n:.3e}  {k}")
    ok &= nbad == 0
    print(f"[model] {'PASS' if ok else 'FAIL'}", flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
