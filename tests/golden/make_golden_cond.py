"""Generates tests/golden/cond_input.npz with the reference's own conditioning path (pytorch/wavenet.py:57-70,190-202:
WaveNet.upsample, WaveNet.cond_layers, WaveNet.get_cond_input) on the CPU, and the permute
pytorch/nv_wavenet.py applies before calling the kernel ([2R][B][L][N] -> [N][L][B][2R]).
The tests only read the committed .npz (kept under 1 MB); regenerating it needs a checkout of the reference project:

    NV_WAVENET_REF=<reference checkout> python tests/golden/make_golden_cond.py
"""
import os
import sys
import warnings

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.environ["NV_WAVENET_REF"], "pytorch"))
warnings.simplefilter("ignore")
import wavenet as ref_wavenet  # noqa: E402  (the reference's module)

out = {}
#        name   C   T  window stride  L   R   B
cases = [("a", 4, 2, 800, 200, 2, 16, 2),         # the reference's upsampling geometry (config.json: window 800, stride 200), 4 bands to keep the file small
         ("b", 5, 7, 12, 4, 3, 4, 3),             # odd small geometry: window = 3 strides
         ("c", 6, 2, 40, 10, 4, 64, 19)]          # R = 64 (the tensor-core / latency kernels' tiled fp16 layouts), two 16-utterance tiles, ragged
for name, C, T, window, stride, L, R, B in cases:
    torch.manual_seed(1234 + C)
    m = ref_wavenet.WaveNet(n_in_channels=256, n_layers=L, max_dilation=2, n_residual_channels=R, n_skip_channels=16,
                            n_out_channels=256, n_cond_channels=C, upsamp_window=window, upsamp_stride=stride)
    feats = torch.randn(B, C, T)
    with torch.no_grad():
        cond = m.get_cond_input(feats)                                  # [2R][B][L][N]
        lh = cond.permute(3, 2, 1, 0).contiguous()                      # [N][L][B][2R], what the kernel consumes
    out.update({f"{name}_features": feats.numpy(), f"{name}_upsample_weight": m.upsample.weight.detach().numpy(),
                f"{name}_upsample_bias": m.upsample.bias.detach().numpy(),
                f"{name}_cond_weight": m.cond_layers.conv.weight.detach().numpy()[:, :, 0],
                f"{name}_cond_bias": m.cond_layers.conv.bias.detach().numpy(), f"{name}_Lh": lh.numpy(),
                f"{name}_geometry": np.array([C, T, window, stride, L, R, B])})
    print(name, tuple(lh.shape), float(lh.abs().max()))
np.savez_compressed(os.path.join(os.path.dirname(__file__), "cond_input.npz"), **out)
