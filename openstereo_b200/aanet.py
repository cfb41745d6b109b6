"""AANet's deformable bottlenecks on the library (aanet/submodule.py:273-410): DeformBottleneck (feature extractor layer3) and
DeformSimpleBottleneck (the deformable aggregation fusions) share one forward,

    out = relu(bn1(conv1(x)));  out = relu(bn2(conv2(out)));  out = bn3(conv3(out));  relu(out + downsample(x) or x)

with conv2 a DeformConv2d: offset_mask = offset_conv(out), offsets = its first dg*18 channels, mask = 2 * sigmoid(the last dg*9)
(double_mask), then the reference's DCNv2 extension.  DeformBottleneckEngine runs conv2 -> bn2 -> relu as ONE launch of the
tensor-core gather mode (ops.mdconv2d_k3_tc, DESIGN.md section 4.21): it reads the offsets and mask logits straight from the raw
offset_conv output and applies 2 * sigmoid as it loads, with bn2 folded into the epilogue.  conv1 / bn1, offset_conv, conv3 / bn3,
downsample and the residual ReLU are the module's own layers.  Parameters stay in the module; the packed weight and the folded BN
are rebuilt when they change.

patch() does not install the engine: on an H100 the gather mode is slower than the reference's own DCNv2 extension, which an AANet
model needs in order to be built at all (DESIGN.md section 4.21).  It serves callers that run a block's forward through it
directly, e.g. ``block.forward = DeformBottleneckEngine(block)`` for CUDA inference, and the tests that pin the gather mode.
"""
import torch

from . import ops


class DeformBottleneckEngine:
    """forward(x) of one DeformBottleneck / DeformSimpleBottleneck (module docstring).  serves(x): the calls the gather mode
    implements -- fp32 input, a modulated 3x3 DeformConv2d with groups = 1, double_mask, an eval-mode BatchNorm2d bn2, Cin a
    multiple of 16 with a multiple of 4 channels per deformable group, Cout in {16, 32, 64, 128}, stride 1 or 2; the module's
    own forward runs every other call."""

    def __init__(self, block):
        self.block = block
        self._key = None
        self._w = self._scale = self._shift = None

    def serves(self, x):
        conv = self.block.conv2
        dc = getattr(conv, "deform_conv", None)
        if x.dtype != torch.float32 or not getattr(conv, "modulation", False) or not getattr(conv, "double_mask", False):
            return False
        if dc is None or dc.groups != 1 or tuple(dc.kernel_size) != (3, 3) or not isinstance(self.block.bn2, torch.nn.BatchNorm2d):
            return False
        stride, dg = _first(dc.stride), dc.deformable_groups
        cin, cout = dc.in_channels, dc.out_channels
        return (ops.mdconv_packed_rows(cout) is not None and cin % 16 == 0 and stride in (1, 2) and cin % dg == 0
                and (cin // dg) % 4 == 0 and not self.block.bn2.training)

    def _ensure(self):
        dc, bn = self.block.conv2.deform_conv, self.block.bn2
        params = [dc.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var] + ([dc.bias] if dc.bias is not None else [])
        key = tuple((t.data_ptr(), t._version) for t in params)
        if key != self._key:
            self._w = ops.pack_tc_weight_2d(dc.weight, 16, pad_cout_to=ops.mdconv_packed_rows(dc.out_channels))
            self._scale, self._shift = ops.fold_bn(bn)
            if dc.bias is not None:
                self._shift = (self._shift + dc.bias.detach().float() * self._scale).contiguous()
            self._key = key

    def __call__(self, x):
        b = self.block
        conv, dc = b.conv2, b.conv2.deform_conv
        self._ensure()
        mon = ops.TcOverflowMonitor.get(x.device)
        mon.check()
        out = b.relu(b.bn1(b.conv1(x)))
        om = conv.offset_conv(out).contiguous()                       # (B, dg*27, Ho, Wo): offsets, then mask logits
        dg = dc.deformable_groups
        out = ops.mdconv2d_k3_tc(out.permute(0, 2, 3, 1).contiguous(), om[:, :dg * 18], om[:, dg * 18:], self._w, self._scale,
                                 self._shift, _first(dc.stride), _first(dc.padding), _first(dc.dilation), dg, ops.ACT_RELU,
                                 ops.MASK_DOUBLE_SIGMOID)
        mon.poll()
        out = b.bn3(b.conv3(out))
        identity = b.downsample(x) if b.downsample is not None else x
        out += identity
        return b.relu(out)


def _first(v):
    return int(v[0]) if isinstance(v, (tuple, list)) else int(v)
