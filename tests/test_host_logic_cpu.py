"""CPU: host-side logic of the product that needs no GPU -- operand packing for the tensor-core kernels (the 3xFP16 split must
be exact), BN folding, the BN-folded backbone twins, state_dict compatibility of the host mirrors, and the gates that keep
CPU tensors away from the CUDA-only paths."""
import pytest
import torch
import torch.nn.functional as F

from openstereo_b200 import host_models as hm
from openstereo_b200 import ops


def rnd(seed, *shape, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


@pytest.mark.parametrize("kc,order", [(32, (0, 1, 2)), (16, (0, 1, 2)), (16, (1, 0, 2)), (16, (1, 2, 0))])
def test_pack_tc_weight_split(kc, order):
    """3xFP16 weight packing: per output channel a power-of-two scale puts max |w| into [2^14, 2^15) (no fp16 overflow, exact to
    undo), hi = nearest fp16, lo = nearest fp16 of the remainder; hi + lo reproduces the scaled weight to 2^-22 relative (2^-25
    absolute once lo is subnormal) with no sign preference, and `inv` is the exact inverse scale times 2^-4 (activation scale)."""
    cout, cin = 8, 64
    w = rnd(1, cout, cin, 3, 3, 3) * torch.logspace(-2, 2, cin).view(1, cin, 1, 1, 1)      # wide dynamic range
    w = w * torch.logspace(-6, 6, cout).view(cout, 1, 1, 1, 1)                               # and very different channel magnitudes
    p = ops.pack_tc_weight(w, kc, kw_order=order)
    assert isinstance(p, ops.TcWeight) and p.kc == kc and p.cout == cout
    assert p.data.shape == (3, cin // kc, 3, 3 * cout, 2 * kc) and p.data.is_contiguous() and p.data.dtype == torch.float16
    assert torch.isfinite(p.data.float()).all()
    # undo the wgmma pre-swizzle (16-byte chunk c of row n is stored at c ^ key(n): an involution), then
    # un-permute: [kd][chunk][kh][kw*cout + co][half*kc + ci] -> (half, co, ci, kd, kh, kw) in the requested kw order
    cpr = 2 * kc // 8
    rows = torch.arange(3 * cout)
    key = (rows & 7) if kc == 32 else ((rows >> 1) & 3)
    src = (torch.arange(cpr).view(1, cpr) ^ key.view(-1, 1)).view(1, 1, 1, 3 * cout, cpr, 1).expand(3, cin // kc, 3, 3 * cout, cpr, 8)
    lin = torch.gather(p.data.view(3, cin // kc, 3, 3 * cout, cpr, 8), 4, src).reshape(3, cin // kc, 3, 3 * cout, 2 * kc)
    assert not torch.equal(lin, p.data)                                                       # the swizzle really moved chunks
    t = lin.double().view(3, cin // kc, 3, 3, cout, 2, kc).permute(5, 4, 1, 6, 0, 2, 3).reshape(2, cout, cin, 3, 3, 3)
    hi, lo = t[0], t[1]
    scale = 2.0 ** -ops.TC_ACT_SCALE_LOG2 / p.inv.double()                                  # 2^e_c
    assert torch.equal(torch.log2(scale), torch.log2(scale).round())                          # exact powers of two
    want = w[..., list(order)].double() * scale.view(-1, 1, 1, 1, 1)
    top = want.abs().amax(dim=(1, 2, 3, 4))
    assert (top >= 2.0 ** 14).all() and (top < 2.0 ** 15).all()
    resid = hi + lo - want
    assert (resid.abs() <= torch.maximum(want.abs() * 2.0 ** -22, torch.tensor(2.0 ** -25, dtype=torch.float64))).all()
    assert abs((resid * want.sign()).sum().item()) <= 0.05 * resid.abs().sum().item()     # zero-mean, not a shrink
    assert ((hi - want).abs() <= want.abs() * 2.0 ** -11).all()                            # round to nearest
    # eff_scale folds the BN scale and is cached per scale tensor
    bn = torch.rand(cout) + 0.5
    assert torch.equal(p.eff_scale(bn), bn * p.inv) and p.eff_scale(bn) is p.eff_scale(bn)
    assert torch.equal(p.eff_scale(None), p.inv)


def test_f16_split_small_and_zero_channels():
    hi, lo = ops.f16_split(torch.tensor([0.0, 1e-6, 1.0, 1000.123, -32767.9]))
    assert torch.isfinite(hi.float()).all() and hi[0] == 0 and lo[0] == 0
    p = ops.pack_tc_weight(torch.zeros(4, 32, 3, 3, 3), 32)                                 # an all-zero channel must not produce inf/nan
    assert torch.isfinite(p.inv).all() and (p.data == 0).all()


def test_pack_deconv_and_head_weights():
    w = rnd(2, 32, 16, 3, 3, 3)                                              # ConvTranspose3d layout (Cin, Cout, ...)
    p = ops.pack_tc_deconv_weight(w)
    assert p.data.shape == (3, 2, 3, 3 * 16, 2 * 16)
    q = ops.pack_tc_weight(w.permute(1, 0, 2, 3, 4).contiguous(), 16, kw_order=(1, 2, 0))
    assert torch.equal(p.data, q.data) and torch.equal(p.inv, q.inv)
    head = rnd(3, 1, 32, 3, 3, 3)
    taps = ops.pack_c1_weight(head)
    assert taps.shape == (27, 32) and torch.equal(taps[(1 * 3 + 2) * 3 + 0], head[0, :, 1, 2, 0])
    with pytest.raises(AssertionError):
        ops.pack_c1_weight(rnd(4, 2, 32, 3, 3, 3))


def test_fold_bn_matches_batch_norm():
    bn = torch.nn.BatchNorm3d(6).eval()
    with torch.no_grad():
        bn.running_mean.copy_(rnd(5, 6)), bn.running_var.copy_(rnd(6, 6).abs() + 0.3)
        bn.weight.copy_(rnd(7, 6)), bn.bias.copy_(rnd(8, 6))
    x = rnd(9, 2, 6, 3, 4, 5)
    scale, shift = ops.fold_bn(bn)
    want = bn(x)
    got = x * scale.view(1, -1, 1, 1, 1) + shift.view(1, -1, 1, 1, 1)
    assert torch.allclose(got, want, rtol=1e-6, atol=1e-6)


def test_folded_backbones_equal_the_originals():
    torch.manual_seed(3)
    for net, x, run in ((hm._GwcFeatureExtraction(True, 12).eval(), rnd(10, 1, 3, 64, 96), lambda m, x: m(x)["gwc_feature"]),
                        (hm._PsmBackbone().eval(), rnd(11, 1, 3, 256, 256), lambda m, x: m._forward(x))):
        with torch.no_grad():
            for mod in net.modules():
                if isinstance(mod, torch.nn.BatchNorm2d):
                    mod.running_mean.normal_(0, 0.2), mod.running_var.uniform_(0.5, 1.5)
                    mod.weight.uniform_(0.5, 1.5), mod.bias.normal_(0, 0.2)
            folded = hm._fold_conv_bn(net)
            assert folded._osb_folded and not any(isinstance(m, torch.nn.BatchNorm2d) for m in folded.modules())
            assert list(net.state_dict().keys())                              # the original keeps its parameters
            a, b = run(net, x), run(folded, x)
            assert ((a - b).abs().max() / a.abs().max()).item() <= 1e-5
            # CPU tensors never take the CUDA-only tensor-core routes
            assert not hm._front_tc_ok(folded, rnd(12, 1, 3, 256, 64))
            assert not hm._lastconv_tc_ok(folded, rnd(13, 1, 320, 8, 128))


def test_geo_class_refuses_cpu_tensors():
    from openstereo_b200 import geo
    with pytest.raises(RuntimeError, match="CUDA tensors required"):
        geo.CombinedGeoEncodingVolume(rnd(14, 1, 4, 2, 8), rnd(15, 1, 4, 2, 8), rnd(16, 1, 2, 6, 2, 8))
    assert geo.Combined_Geo_Encoding_Volume is geo.CombinedGeoEncodingVolume


def test_host_mirror_state_dict_keys_match_the_oracle_models():
    """host_models mirrors load reference checkpoints: same keys (and shapes) as the oracle models, whose keys are asserted
    equal to the reference's in tools/make_golden.py."""
    from oracle import models as omodels
    cfg = {"MAX_DISP": 192, "USE_CONCAT_VOLUME": True, "CONCAT_CHANNELS": 12, "DOWNSAMPLE": 4, "NUM_GROUPS": 40}
    mine, ref = hm.GwcNet(cfg), omodels.GwcNet(192, True, 12, 4, 40)
    assert {k: tuple(v.shape) for k, v in mine.state_dict().items()} == {k: tuple(v.shape) for k, v in ref.state_dict().items()}
    mine, ref = hm.PSMNet({"MAX_DISP": 192}), omodels.PSMNet(192)
    assert {k: tuple(v.shape) for k, v in mine.state_dict().items()} == {k: tuple(v.shape) for k, v in ref.state_dict().items()}


def test_packed_layer_refuses_unsupported_hyperparameters():
    """ADVICE r1: an engine built from a module tree that deviates from the reference architectures must not silently compute a
    different convolution (the kernels hard-wire padding k//2, dilation 1, groups 1, the two transposed-conv flavours)."""
    import torch.nn as nn
    from openstereo_b200 import aggregation as agg
    for good in (nn.Conv3d(8, 8, 3, 1, 1, bias=False), nn.Conv3d(8, 8, 3, 2, 1), nn.Conv3d(8, 4, 1), nn.Conv2d(8, 8, 1),
                 nn.ConvTranspose3d(8, 8, 3, 2, 1, 1, bias=False), nn.ConvTranspose3d(8, 8, 4, 2, 1, bias=False)):
        agg._Packed(good)
    for bad in (nn.Conv3d(8, 8, 3, 1, 2, dilation=2), nn.Conv3d(8, 8, 3, 1, 1, groups=2), nn.Conv3d(8, 8, (3, 1, 1), 1, (1, 0, 0)),
                nn.Conv3d(8, 8, 3, 1, 0), nn.Conv3d(8, 8, 5, 1, 2), nn.ConvTranspose3d(8, 8, 3, 2, 1, 0), nn.ConvTranspose3d(8, 8, 4, 2, 0)):
        with pytest.raises(NotImplementedError):
            agg._Packed(bad)


def test_pack_tc_weight_k4_transposed():
    """ConvTranspose3d(k4) packing for conv3d_tcdc<KS = 4>: [4 kd][chunks][4 kh][4 * Cout (kw order 1, 3, 2, 0)][16 hi | 16 lo]."""
    cin, cout = 32, 16
    w = rnd(5, cin, cout, 4, 4, 4)
    p = ops.pack_tc_deconv_weight(w)
    assert p.ksize == 4 and p.kc == 16 and p.cout == cout
    assert p.data.shape == (4, cin // 16, 4, 4 * cout, 32) and p.data.dtype == torch.float16 and p.data.is_contiguous()
    cpr = 4
    rows = torch.arange(4 * cout)
    key = (rows >> 1) & 3
    src = (torch.arange(cpr).view(1, cpr) ^ key.view(-1, 1)).view(1, 1, 1, 4 * cout, cpr, 1).expand(4, cin // 16, 4, 4 * cout, cpr, 8)
    lin = torch.gather(p.data.view(4, cin // 16, 4, 4 * cout, cpr, 8), 4, src).reshape(4, cin // 16, 4, 4 * cout, 32)
    t = lin.double().view(4, cin // 16, 4, 4, cout, 2, 16).permute(5, 4, 1, 6, 0, 2, 3).reshape(2, cout, cin, 4, 4, 4)
    scale = 2.0 ** -ops.TC_ACT_SCALE_LOG2 / p.inv.double()
    want = w.permute(1, 0, 2, 3, 4)[..., [1, 3, 2, 0]].double() * scale.view(-1, 1, 1, 1, 1)
    assert ((t[0] + t[1] - want).abs() <= torch.maximum(want.abs() * 2.0 ** -22, torch.tensor(2.0 ** -25, dtype=torch.float64))).all()
    p3 = ops.pack_tc_deconv_weight(rnd(6, cin, cout, 3, 3, 3))                               # the k3 packing is unchanged
    assert p3.ksize == 3 and p3.data.shape == (3, cin // 16, 3, 3 * cout, 32)


def test_tensor_core_capability_queries():
    """Which shapes the tensor-core variants serve (answered by the C library without a GPU): whole-row widths, general widths through
    column tiles (>= OSB_TC_MIN_WIDTH = 24), the StereoBase plan (Cout 96, k4 transposed conv, W' = 16 channel slices)."""
    assert ops.conv3d_tc_kc(32, 32, 128) == 32 and ops.conv3d_tc_kc(64, 64, 64) == 16 and ops.conv3d_tc_kc(128, 128, 32) == 16
    for w in (240, 312, 160, 120, 78, 60, 24):
        assert ops.conv3d_tc_kc(32, 32, w) == 16 and ops.conv3d_tc_kc(128, 128, w) == 16
        assert ops.deconv3d_tc_supported(64, 32, w) and ops.deconv3d_tc_supported(128, 64, w)
        assert ops.conv3d_s2_tc_supported(32, 64, 8, 8, 2 * w)
    assert ops.conv3d_tc_kc(32, 32, 20) == 0 and not ops.deconv3d_tc_supported(64, 32, 20)
    assert ops.conv3d_tc_kc(24, 32, 240) == 0 and ops.conv3d_tc_kc(32, 48, 240) == 0          # channels must be multiples of 16 / known Cout
    assert not ops.conv3d_s2_tc_supported(32, 64, 7, 8, 128)                                  # odd extents have no stride-2 variant
    assert ops.conv3d_tc_kc(96, 96, 32) == 16 and ops.conv3d_s2_tc_supported(64, 96, 8, 8, 64)
    assert ops.deconv3d_k4_tc_supported(96, 64, 32) and ops.deconv3d_k4_tc_supported(64, 32, 64)
    assert ops.conv3d_tc_kc(160, 96, 16) == 16 and ops.conv3d_tc_kc(160, 64, 16) == 16 and ops.deconv3d_k4_tc_supported(160, 32, 16)
    assert not ops.deconv3d_k4_tc_supported(96, 96, 16) and not ops.deconv3d_k4_tc_supported(24, 32, 64)


def test_stereobase_tc_route_gating_without_gpu():
    """StereoBaseAggregation.tc_route_ok: shape / channel-plan gates of the tensor-core route (pure host logic)."""
    from openstereo_b200 import aggregation as agg
    from oracle import aggregation as oagg
    m = oagg.StereoBaseHourglass(24, [96, 64, 192, 160]).eval()
    eng = agg.StereoBaseAggregation(m)
    with torch.no_grad():
        eng._pack()
    assert eng.tc_route_ok((4, 24, 48, 64, 128)) and eng._level32_tc_ok((4, 24, 48, 64, 128))
    assert not eng.tc_route_ok((4, 24, 48, 64, 120)) and not eng.tc_route_ok((4, 24, 44, 64, 128))   # width 120 / D' not a multiple of 8
    assert not eng.tc_route_ok((4, 32, 48, 64, 128))                                                  # not this module's channel plan
    agg.USE_TENSOR_CORES = False
    try:
        assert not eng.tc_route_ok((4, 24, 48, 64, 128))
    finally:
        agg.USE_TENSOR_CORES = True


def _launcher_variants():
    """Every launch_tc / launch_tcg / launch_tcs2 / launch_tcdc template list the selectors in csrc/ name, with the launcher's
    default template arguments filled in, in the spelling of osb_tc_last_variant() ("tcg<64,16,64,1,1,0,1>")."""
    import glob
    import os
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = "".join(open(p).read() for p in sorted(glob.glob(os.path.join(root, "openstereo_b200", "csrc", "*.cu"))))
    lit = {"true": "1", "false": "0"}
    defaults = {}
    for params, name in re.findall(r"template\s*<([^<>]*)>\s*(?:static\s+)?int\s+(launch_tc\w*)\s*\(", src):
        defaults[name] = [p.split("=")[1].strip() if "=" in p else None for p in params.split(",")]
    assert set(defaults) == {"launch_tc", "launch_tcg", "launch_tcs2", "launch_tcdc"}, sorted(defaults)
    found = set()
    for name, args in re.findall(r"\b(launch_tc\w*)<([^<>]*)>", src):
        vals = [a.strip() for a in args.split(",")]
        vals += defaults[name][len(vals):]
        assert None not in vals, (name, args)
        found.add("%s<%s>" % (name[len("launch_"):], ",".join(lit.get(v, v) for v in vals)))
    return found


def test_tc_contract_registry_matches_selectors():
    """A tensor-core instantiation cannot land without a row in the contract registry of tests/test_tc_contract_gpu.py (routing,
    grid-cap, per-channel accuracy, store-bounds, range-guard and kappa . n checks), and no row may name one that is gone."""
    from test_tc_contract_gpu import REGISTRY
    found = _launcher_variants()
    rows = {r.variant for r in REGISTRY}
    assert not found - rows, "instantiations without a contract row: %s" % sorted(found - rows)
    assert not rows - found, "contract rows naming no instantiation: %s" % sorted(rows - found)


# flavours.cu kernels that are not convolutions: volume / regression gathers and reductions with their own oracle tests
_NOT_CONVOLUTIONS = {"group_l2_normalize_kernel", "sub_volume_kernel", "regression_values_kernel"}
# the local `auto kernel = ...<template parameters>` of each templated launcher, covered by the launcher's template lists
_TEMPLATED_LAUNCHERS = {"conv3d_k3_kernel": "launch_conv_k3", "deconv3d_kernel": "launch_deconv",
                        "conv1x1_ndhwc_cat_kernel": "launch_conv1x1_cat", "mbv2_block3d_kernel": "launch_mbv2"}


def _cuda_core_variants():
    """Every launch_conv_k3 / launch_deconv / launch_conv1x1_cat / launch_mbv2 template list and every kernel launched directly
    with <<< in the CUDA-core convolution sources, in the registry spelling ("launch_deconv<3,8>", "conv1x1_ndhwc_kernel<64,64>")."""
    import os
    import re
    csrc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "openstereo_b200", "csrc")
    found = set()
    for name in ("conv3d.cu", "lightstereo.cu", "msnet.cu", "flavours.cu"):
        src = open(os.path.join(csrc, name)).read()
        for launcher, args in re.findall(r"\b(launch_conv_k3|launch_deconv|launch_conv1x1_cat|launch_mbv2)\s*<([^<>]*)>", src):
            found.add("%s<%s>" % (launcher, args.replace(" ", "")))
        for m in re.finditer(r"\b(\w+)\s*(<[^<>]*>)?\s*<<<", src):
            kernel, args = m.group(1), (m.group(2) or "").replace(" ", "")
            if kernel == "kernel":                               # auto kernel = name<args>; ... kernel<<<...>>>
                kernel, args = re.findall(r"auto\s+kernel\s*=\s*(\w+)\s*(<[^<>]*>)?\s*;", src[:m.start()])[-1]
                args = args.replace(" ", "")
                if not re.fullmatch(r"(<\d+(,\d+)*>)?", args):
                    assert kernel in _TEMPLATED_LAUNCHERS, "%s: %s%s launched from an unknown templated launcher" % (name, kernel, args)
                    continue
            if kernel not in _NOT_CONVOLUTIONS:
                found.add(kernel + args)
    return found


def test_cuda_core_contract_registry_matches_sources():
    """A CUDA-core convolution instantiation or launch path cannot land without a row in the contract registry of
    tests/test_cuda_core_contract_gpu.py (routing, per-channel accuracy, both store paths, store bounds, determinism, grid caps),
    and no row may name one that is gone."""
    from test_cuda_core_contract_gpu import REGISTRY
    found = _cuda_core_variants()
    rows = {r.variant for r in REGISTRY}
    assert not found - rows, "instantiations without a contract row: %s" % sorted(found - rows)
    assert not rows - found, "contract rows naming no instantiation: %s" % sorted(rows - found)


# Files of the non-convolution kernels.  Two __global__ functions there have rows in the convolution registries instead.
_KERNEL_CONTRACT_FILES = ("volume.cu", "softargmin.cu", "backward.cu", "geo.cu", "cascade.cu", "coex.cu", "flavours.cu", "conv3d_tc.cu")
_CONVOLUTIONS_THERE = {"feature_att_gate_kernel", "conv3d_tc_kernel"}
_GLOBAL = r"__global__\s+void\s+(?:__launch_bounds__\s*\([^()]*\)\s*)?(\w+)\s*\("


def _csrc(name):
    import os
    import re
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "openstereo_b200", "csrc", name)
    return re.sub(r'//[^\n]*|/\*.*?\*/|"(?:\\.|[^"\\\n])*"', "", open(path).read(), flags=re.S)   # code only: no comments, no strings


def _kernel_contract_variants():
    """Every __global__ instantiation the non-convolution sources can launch, in the registry spelling ("volume_kernel<true,false>",
    "coex_regression_kernel<5>", "softargmin_kernel").  A templated kernel contributes each spelling with literal template
    arguments: the function-pointer table of launch_volume, the ternary of launch_warped, the switch of osb_coex_regression_fwd,
    the if / else of osb_geo_lookup_fwd and direct <<< launches.  An untemplated kernel must be launched with <<<."""
    import re
    found = set()
    for name in _KERNEL_CONTRACT_FILES:
        src = _csrc(name)
        for kernel in set(re.findall(_GLOBAL, src)) - _CONVOLUTIONS_THERE:
            if re.search(r"template\s*<[^<>]*>\s*" + _GLOBAL.replace(r"(\w+)", kernel), src):
                spellings = re.findall(r"\b%s\s*<([^<>;()]*)>" % kernel, src)
                assert spellings, "%s: templated %s has no instantiation" % (name, kernel)
                for args in spellings:
                    args = args.replace(" ", "").replace("\n", "")
                    assert re.fullmatch(r"(true|false|\d+)(,(true|false|\d+))*", args), "%s: %s<%s> is not literal" % (name, kernel, args)
                    found.add("%s<%s>" % (kernel, args))
            else:
                assert re.search(r"\b%s\s*<<<" % kernel, src), "%s: %s is never launched with <<<" % (name, kernel)
                found.add(kernel)
    return found


def test_kernel_contract_registry_matches_sources():
    """A cost-volume, regression, lookup, backward or layout kernel cannot land without a row in the contract registry of
    tests/test_kernel_contract_gpu.py (routing, accuracy against fp64, store bounds, store paths, determinism), and no row may
    name one that is gone.  With the two convolution registries, every __global__ function defined under csrc/ has a row."""
    import glob
    import os
    import re
    from test_cuda_core_contract_gpu import REGISTRY as CUDA_CORE, kernel_of
    from test_kernel_contract_gpu import REGISTRY
    from test_tc_contract_gpu import REGISTRY as TENSOR_CORE
    found = _kernel_contract_variants()
    assert {"volume_kernel<false,false>", "volume_kernel<true,true>", "warped_volume_kernel<16>", "coex_regression_kernel<8>",
            "geo_lookup_kernel<0>", "upsample_softargmin_kernel<true>", "ncdhw_to_ndhwc_kernel"} <= found
    rows = {r.variant for r in REGISTRY}
    assert not found - rows, "instantiations without a contract row: %s" % sorted(found - rows)
    assert not rows - found, "contract rows naming no instantiation: %s" % sorted(rows - found)
    covered = {v.split("<")[0] for v in rows}
    covered |= {kernel_of(r.variant).split("<")[0] for r in CUDA_CORE}
    covered |= {"conv3d_%s_kernel" % r.variant.split("<")[0] for r in TENSOR_CORE}
    defined = set()
    for path in glob.glob(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "openstereo_b200", "csrc", "*.cu*")):
        defined |= set(re.findall(_GLOBAL, _csrc(os.path.basename(path))))
    assert len(defined) >= 30
    assert not defined - covered, "__global__ functions with no row in any contract registry: %s" % sorted(defined - covered)
