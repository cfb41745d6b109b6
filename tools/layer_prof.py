#!/usr/bin/env python
"""Run ONE aggregation layer at its bench shape (channels-last in/out) a few times: the target of ncu captures and of quick
per-layer timings.  usage: layer_prof.py <stem|conv2|conv4|conv1s2|conv3s2|conv5|conv6|bb64|bb2e|ds2|...> [batch] [iters]
OSB_LP_SPLIT=1: the W = 128 stride-1 layers (stem, stem64, stem64n, head) read and write split activations (ops.to_split), as
GwcNet's stem chain does; the input is converted once, outside the timed calls.
OSB_LP_CUDNN=1: the 2D backbone layers (bb*, ds*) run as the module's own NCHW Conv2d on cuDNN instead (fp32, TF32 off, algorithm
search on, as bench.py runs it)."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from openstereo_b200 import ops  # noqa: E402
from tools.kbench import timeit  # noqa: E402

LAYERS = {  # name: (kind, cin, cout, D, H, W of the INPUT)
    "stem": ("s1", 32, 32, 48, 64, 128), "stem64": ("s1", 64, 32, 48, 64, 128), "stem64n": ("s1n", 64, 32, 48, 64, 128),
    "head": ("s1h", 32, 1, 48, 64, 128),
    # 2D backbone residual-block convs as one-plane volumes (B = 16 images = 8 pairs): layer2 64->64, layer3 128->128, front 32->32
    "bb64": ("2d", 64, 64, 1, 64, 128), "bb128": ("2d", 128, 128, 1, 64, 128), "bb32": ("2d", 32, 32, 1, 256, 128),
    # stage entries: layer2[0].conv1 (stride 2, one-plane stride-2 conv), layer3[0].conv1 (64->128), their 1x1 downsamples (fp32
    # pointwise kernel on the NCHW input; the stride-2 one includes the copy of the even rows and columns)
    "bb2e": ("2ds2", 32, 64, 1, 128, 256), "bb3e": ("2d", 64, 128, 1, 64, 128),
    "ds2": ("1x1s2", 32, 64, 1, 128, 256), "ds3": ("1x1", 64, 128, 1, 64, 128),
    "conv2": ("s1", 64, 64, 24, 32, 64), "conv4": ("s1", 128, 128, 12, 16, 32),
    "conv1s2": ("s2", 32, 64, 48, 64, 128), "conv3s2": ("s2", 64, 128, 24, 32, 64),
    "conv5": ("dc", 128, 64, 12, 16, 32), "conv6": ("dc", 64, 32, 24, 32, 64),
}


def main():
    name = sys.argv[1]
    B = int(sys.argv[2]) if len(sys.argv) > 2 else 8
    iters = int(sys.argv[3]) if len(sys.argv) > 3 else 5
    kind, cin, cout, d, h, w = LAYERS[name]
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(B, d, h, w, cin, device=dev, generator=g)
    sc, sh = torch.rand(cout, device=dev, generator=g) + 0.5, torch.randn(cout, device=dev, generator=g) * 0.1
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=dev)
    split = bool(os.environ.get("OSB_LP_SPLIT")) and kind in ("s1", "s1n", "s1h") and w == 128
    if kind in ("2d", "2ds2", "1x1", "1x1s2"):
        B, s, k = 2 * B, 2 if kind.endswith("s2") else 1, 1 if kind.startswith("1x1") else 3
        macs = B * (h // s) * (w // s) * k * k * cin * cout
        wgt = torch.randn(cout, cin, k, k, device=dev, generator=g) * 0.05
        xn = torch.randn(B, cin, h, w, device=dev, generator=g)
    if os.environ.get("OSB_LP_CUDNN") and kind in ("2d", "2ds2", "1x1", "1x1s2"):
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cudnn.benchmark = True
        fn = lambda: torch.nn.functional.conv2d(xn, wgt, sh, s, k // 2)  # noqa: E731
    elif kind == "2ds2":
        w5 = torch.zeros(cout, cin, 3, 3, 3, device=dev)
        w5[:, :, 1] = wgt
        wp = ops.pack_tc_weight(w5, 16, kw_order=(1, 0, 2))
        x = torch.randn(B, 1, h, w, cin, device=dev, generator=g)
        fn = lambda: ops.conv3d_k3_s2_tc(x, wp, None, sh, None, ops.ACT_RELU, out_ndhwc=True)  # noqa: E731
    elif kind in ("1x1", "1x1s2"):
        wp = ops.pack_conv_weight(wgt.unsqueeze(2))
        fn = lambda: ops.conv3d_1x1(xn[:, :, ::s, ::s].contiguous(), wp, None, sh)  # noqa: E731
    elif kind == "2d":
        x = torch.randn(B, h, w, cin, device=dev, generator=g)
        w5 = torch.zeros(cout, cin, 3, 3, 3, device=dev)
        w5[:, :, 1] = wgt
        wp = ops.pack_tc_weight(w5, ops.conv2d_tc_kc(cin, cout, w, 1))
        res = None if os.environ.get("OSB_LP_NORES") else torch.randn(B, h, w, cout, device=dev, generator=g)
        fn = lambda: ops.conv2d_k3_tc(x, wp, None, sh, res, ops.ACT_RELU)  # noqa: E731
    elif kind == "dc":
        wgt = torch.randn(cin, cout, 3, 3, 3, device=dev, generator=g) * 0.05
        wp = ops.pack_tc_deconv_weight(wgt)
        res = None if os.environ.get("OSB_LP_NORES") else torch.randn(B, 2 * d, 2 * h, 2 * w, cout, device=dev, generator=g)
        fn = lambda: ops.deconv3d_k3_tc(x, wp, sc, sh, res, ops.ACT_RELU, out_ndhwc=True, res_ndhwc=True)  # noqa: E731
        macs = B * d * h * w * 27 * cin * cout
    elif kind == "s2":
        wgt = torch.randn(cout, cin, 3, 3, 3, device=dev, generator=g) * 0.05
        wp = ops.pack_tc_weight(wgt, 16, kw_order=(1, 0, 2))
        fn = lambda: ops.conv3d_k3_s2_tc(x, wp, sc, sh, None, ops.ACT_RELU, out_ndhwc=True)  # noqa: E731
        macs = B * (d // 2) * (h // 2) * (w // 2) * 27 * cin * cout
    elif kind == "s1n":                                        # NCDHW input (the cost volume as the volume kernel wrote it)
        wgt = torch.randn(cout, cin, 3, 3, 3, device=dev, generator=g) * 0.05
        wp = ops.pack_tc_weight(wgt, ops.conv3d_tc_kc(cin, cout, w))
        xn = x.permute(0, 4, 1, 2, 3).contiguous()
        fn = lambda: ops.conv3d_k3_tc(xn, wp, sc, sh, None, ops.ACT_RELU, out_ndhwc=True, in_ncdhw=True, out_split=split)  # noqa: E731
        macs = B * d * h * w * 27 * cin * cout
    elif kind == "s1h":                                        # 32 -> 1 classifier head on the narrow variant
        wgt = torch.randn(cout, cin, 3, 3, 3, device=dev, generator=g) * 0.05
        wp = ops.pack_tc_weight(wgt, 32, pad_cout_to=16)
        x = ops.to_split(x.permute(0, 4, 1, 2, 3).contiguous()) if split else x
        fn = lambda: ops.conv3d_k3_tc(x, wp, None, None, None, ops.ACT_NONE, out_ndhwc=False, res_ndhwc=False)  # noqa: E731
        macs = B * d * h * w * 27 * cin * cout
    else:
        wgt = torch.randn(cout, cin, 3, 3, 3, device=dev, generator=g) * 0.05
        wp = ops.pack_tc_weight(wgt, ops.conv3d_tc_kc(cin, cout, w))
        x = ops.to_split(x.permute(0, 4, 1, 2, 3).contiguous()) if split else x
        fn = lambda: ops.conv3d_k3_tc(x, wp, sc, sh, None, ops.ACT_RELU, out_ndhwc=True, out_split=split)  # noqa: E731
        macs = B * d * h * w * 27 * cin * cout
    ms, _ = timeit(fn, iters, flush)
    print(json.dumps({"layer": name, "split": split, "cudnn": bool(os.environ.get("OSB_LP_CUDNN")), "ms": round(ms, 4), "useful_TF": round(2 * macs / ms / 1e9, 1)}), flush=True)


if __name__ == "__main__":
    main()
