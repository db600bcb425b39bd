"""Forward-only timing of the hybrid ResNet-lite stem at merlot.yaml's sizes (32 frames 192x352, resnet_layers [3,4,9]):
CUDA-event time of lite_resnet50 + conv_postresnet_proj inside the model's forward helper, vs the 433 GFLOP of SURVEY Appendix D."""
import sys

import torch

sys.path.insert(0, ".")
import bench  # noqa: E402
from merlot_b200.modeling import MerlotModel  # noqa: E402
from merlot_b200.params import ParamStore  # noqa: E402
from merlot_b200.train import synthetic_batch  # noqa: E402

cfg = bench.load_config()
cfg.model["resnet_layers"] = [3, 4, 9]
store = ParamStore(cfg.model, device="cuda", with_optimizer_state=False)
store.init_reference(seed=0)
feats = synthetic_batch(cfg, bench.PER_GPU_BATCH, seed=0)
m = MerlotModel(config=cfg.model, is_training=False, image=feats["images"], input_ids=feats["input_ids"], use_tpu=False,
                shuffled_idx_img=feats["shuffled_idx_img"], mask_input=False, params=store)
torch.cuda.synchronize()
img = feats["images"].contiguous()
N = img.shape[0]
for _ in range(2):
    rc, h, w = m._stem.forward(img, N, 192, 352)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(5):
    rc, h, w = m._stem.forward(img, N, 192, 352)
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / 5
print(f"hybrid stem forward: {ms:.2f} ms for {N} frames -> [{N}x{h}x{w}, {rc.shape[1]}]; 432.8 GFLOP => {432.8 / ms:.0f} TFLOP/s; "
      f"finite={bool(torch.isfinite(rc.float()).all())} mean|x|={rc.float().abs().mean().item():.3f}")
