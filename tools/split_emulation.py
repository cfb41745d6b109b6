"""CPU emulation of the 3xTF32 operand split of the tensor-core conv kernels, to measure what a split policy costs in
end-to-end EPE WITHOUT a GPU (round-2 bisect of the 2.27e-3 px failure at 256x512).

Every Conv3d / ConvTranspose3d (and optionally Conv2d) of the oracle GwcNet is replaced by
    conv(a_hi, b_hi) + conv(a_hi, b_lo') + conv(a_lo', b_hi)
with the operands split the way a policy says:
    trunc : hi = x & ~0x1fff, lo = x - hi, lo' = lo & ~0x1fff      (round 1: what the kernels + hardware did)
    rna   : hi = rna_tf32(x),  lo = x - hi, lo' = rna_tf32(lo)      (round 2)
and compared with the plain fp32 oracle.  Usage: python tools/split_emulation.py [--h 256 --w 512] [--conv2d]
"""
import argparse
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import models as omodels          # noqa: E402
from oracle import seeded_init as si          # noqa: E402


def trunc13(x):
    return (x.contiguous().view(torch.int32) & -8192).view(torch.float32)


def rna13(x):
    return ((x.contiguous().view(torch.int32) + 4096) & -8192).view(torch.float32)


def split(x, policy):
    if policy == "trunc":
        hi = trunc13(x)
        return hi, trunc13(x - hi)
    hi = rna13(x)
    return hi, rna13(x - hi)


class Emulate:
    def __init__(self, policy, conv2d=False):
        self.policy, self.conv2d = policy, conv2d

    def __enter__(self):
        self.orig = (F.conv3d, F.conv_transpose3d, F.conv2d)
        pol = self.policy

        def wrap(fn):
            def f(x, w, bias=None, *a, **k):
                xh, xl = split(x, pol)
                wh, wl = split(w, pol)
                y = fn(xl, wh, None, *a, **k) + fn(xh, wl, None, *a, **k)
                y = y + fn(xh, wh, None, *a, **k)
                if bias is not None:
                    y = y + bias.view(1, -1, *([1] * (y.dim() - 2)))
                return y
            return f
        F.conv3d, F.conv_transpose3d = wrap(self.orig[0]), wrap(self.orig[1])
        if self.conv2d:
            F.conv2d = wrap(self.orig[2])
        return self

    def __exit__(self, *exc):
        F.conv3d, F.conv_transpose3d, F.conv2d = self.orig


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--h", type=int, default=256)
    ap.add_argument("--w", type=int, default=512)
    ap.add_argument("--conv2d", action="store_true")
    args = ap.parse_args()
    torch.manual_seed(0)
    model = omodels.GwcNet(192, True, 12, 4, 40).eval()
    model.load_state_dict(si.seeded_state_dict(model.state_dict(), seed=1, scale=si.GWCNET_SCALE))
    g = torch.Generator().manual_seed(0)
    x = {"left": torch.randn(1, 3, args.h, args.w, generator=g), "right": torch.randn(1, 3, args.h, args.w, generator=g)}
    with torch.no_grad():
        want = model(dict(x))["disp_pred"]
        print("fp32 oracle: disp std %.2f" % want.std().item())
        for pol in ("trunc", "rna"):
            with Emulate(pol, args.conv2d):
                got = model(dict(x))["disp_pred"]
            d = (got - want)
            print("%-5s split%s: EPE %.3e px, mean signed %.3e, max %.3e" % (pol, " (+conv2d)" if args.conv2d else "",
                                                                           d.abs().mean().item(), d.mean().item(), d.abs().max().item()))


if __name__ == "__main__":
    main()
