"""Informative same-box baseline: the oracle restatements (stock torch ops: grid_sample, avg_pool2d, conv3d, cuDNN convs)
run on the GPU through PyTorch-CUDA, next to this repo's kernels.  Test/bench infrastructure only."""
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from monorec_b200.model import MonoRecModel  # noqa: E402
from monorec_b200.synthetic import make_inputs, to_device  # noqa: E402
from oracle import convnet_oracle as CO  # noqa: E402
from oracle import cost_volume_oracle as O  # noqa: E402

B, F = 8, 4
dev = "cuda:0"
torch.manual_seed(0)
model = MonoRecModel().to(dev).eval()
sd = {k: v for k, v in model.state_dict().items()}
data = to_device(make_inputs(B, F, 256, 512, seed=0), dev)


def timed(fn, n=3):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


# the oracle's cost volume builds CPU-side constants; move what it needs by running it with CUDA default device
torch.set_default_device(dev)
with torch.no_grad():
    t_cv = timed(lambda: O.cost_volume_torch(data), 2)
    cv, sf = O.cost_volume_torch(data)
    feats = model._feature_extractor(data["keyframe"] + .5)
    for tf32 in (False, True):
        torch.backends.cudnn.allow_tf32 = tf32
        torch.backends.cuda.matmul.allow_tf32 = tf32
        t_mask = timed(lambda: CO.mask_module(sd, sf, feats))
        mask = CO.mask_module(sd, sf, feats)
        t_depth = timed(lambda: CO.depth_module(sd, (1 - mask) * cv, data["keyframe"], feats))
        print(f"torch-CUDA (cudnn tf32={tf32}) B={B}: mask {t_mask:.2f} ms, depth {t_depth:.2f} ms")
print(f"torch-CUDA cost volume (ATen grid_sample/avg_pool/conv3d) B={B}: {t_cv:.2f} ms = {1e3 * B / t_cv:.1f} keyframes/s")
