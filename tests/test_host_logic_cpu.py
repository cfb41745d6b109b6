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


def _struct_fields(name, struct):
    """Field names of `struct <struct> { ... };` in csrc/<name> (member functions skipped, array extents dropped)."""
    import re
    body = re.search(r"struct\s+%s\s*\{(.*?)\n\};" % struct, _csrc(name), re.S).group(1)
    body = re.sub(r"(?:\w+\s+)*[\w:<>]+\s+\w+\s*\([^()]*\)\s*(?:const\s*)?\{[^{}]*\}", "", body)   # __device__ void f() const { }
    fields = []
    for stmt in body.split(";"):
        stmt = re.sub(r"=[^,]*|\[[^\]]*\]", "", stmt).strip()                                # initialisers, [GEO_MAX_LEVELS]
        if stmt:
            fields += [re.findall(r"\w+", part)[-1] for part in stmt.split(",")]
    return fields


def _kernel_params(name, kernel):
    """Parameter names of __global__ <kernel>(...) in csrc/<name>.  A parameter passed by value whose type is a struct defined in
    that file is replaced by its fields, spelled as the kernel reads them ("p.crop", "ad.align")."""
    import re
    src = _csrc(name)
    structs = set(re.findall(r"\bstruct\s+(\w+)\s*\{", src))
    params = re.search(_GLOBAL.replace(r"(\w+)", kernel) + r"([^()]*)\)", src).group(1)
    names = []
    for p in params.split(","):
        words = re.findall(r"\w+", p)
        struct = [w for w in words[:-1] if w in structs]
        if struct and "*" not in p and "&" not in p:
            names += ["%s.%s" % (words[-1], f) for f in _struct_fields(name, struct[0])]
        else:
            names.append(words[-1])
    return names


def test_tc_runtime_modes_have_contract_rows():
    """Every field of struct TcArgs is classified in TC_ARGS_FIELDS (tests/test_tc_contract_gpu.py) as an operand / geometry field or
    as a runtime mode; every mode has its rows: one per instantiation MODE_VARIANTS lists for it (test_mode_sweep checks that list on
    the GPU), and the split rows cover every accepted (input, output, residual) layout combination."""
    from test_tc_contract_gpu import MODE_VARIANTS, REGISTRY, SPLIT_COMBOS, TC_ARGS_FIELDS
    fields = _struct_fields("tc_common.cuh", "TcArgs")
    assert len(fields) == len(set(fields)) and {"x", "terms", "dcn_mask_mode", "res_bstride"} <= set(fields)
    assert set(fields) == set(TC_ARGS_FIELDS), "TcArgs fields not classified: %s; classified fields that are gone: %s" % (
        sorted(set(fields) - set(TC_ARGS_FIELDS)), sorted(set(TC_ARGS_FIELDS) - set(fields)))
    modes = {r.mode for r in REGISTRY} - {""}
    assert {m for m in TC_ARGS_FIELDS.values() if m} <= modes and modes == set(MODE_VARIANTS)
    for mode, variants in MODE_VARIANTS.items():
        rows = [r for r in REGISTRY if r.mode == mode]
        assert {r.variant for r in rows} == variants, "mode %s: instantiations without a row: %s" % (
            mode, sorted(variants - {r.variant for r in rows}))
        if mode != "split":
            assert len({r.variant for r in rows}) == len(rows), "mode %s: two rows for one instantiation" % mode
    assert {r.opt for r in REGISTRY if r.mode == "split"} == SPLIT_COMBOS
    dcn = [r for r in REGISTRY if r.kind == "dcn"]
    assert {r.opt[0] for r in dcn} == {1, 2} and {r.opt[1] for r in dcn} == {1, 2, 3}
    assert {r.cin // r.opt[2] for r in dcn} >= {4, 8, 16}


def _nonconv_kernel_params():
    """{kernel: parameter names} for every __global__ function of the non-convolution sources, by-value structs field by field."""
    import re
    params = {}
    for name in _KERNEL_CONTRACT_FILES:
        for kernel in set(re.findall(_GLOBAL, _csrc(name))) - _CONVOLUTIONS_THERE:
            assert kernel not in params, "%s is defined twice" % kernel
            params[kernel] = _kernel_params(name, kernel)
    return params


def test_nonconv_runtime_modes_have_contract_rows():
    """Every parameter of every __global__ function in the non-convolution sources (a by-value struct such as VolParams, GeoParams,
    WarpParams, RegressionParams or Axis field by field) is classified in NONCONV_KERNEL_PARAMS (tests/test_kernel_contract_gpu.py) as
    an operand / geometry field or as the runtime mode it selects; every mode is one row family whose rows reach exactly the
    instantiations NONCONV_MODE_VARIANTS lists for it (test_routing checks each row's on the GPU), all of them of the kernels whose
    parameters select the mode; each mode's rows meet MODE_REQUIREMENTS; each lookup family has a row whose taps take the fallback
    read and a row at grid z = 65535; both warped_volume_kernel instantiations have a cas row with the left copy unmasked."""
    from test_kernel_contract_gpu import MODE_REQUIREMENTS, NONCONV_KERNEL_PARAMS, NONCONV_MODE_VARIANTS, REGISTRY, grid_z
    found = _nonconv_kernel_params()
    assert set(found) == set(NONCONV_KERNEL_PARAMS), "kernels not classified: %s; classified kernels that are gone: %s" % (
        sorted(set(found) - set(NONCONV_KERNEL_PARAMS)), sorted(set(NONCONV_KERNEL_PARAMS) - set(found)))
    selects = {}                                                        # mode -> kernels with a parameter that selects it
    for kernel, params in found.items():
        table = NONCONV_KERNEL_PARAMS[kernel]
        assert params and len(params) == len(set(params)), (kernel, params)
        assert set(params) == set(table), "%s parameters not classified: %s; classified parameters that are gone: %s" % (
            kernel, sorted(set(params) - set(table)), sorted(set(table) - set(params)))
        for mode in set(table.values()) - {""}:
            selects.setdefault(mode, set()).add(kernel)
    assert {"p.crop", "p.mask_left", "tgt_map"} <= set(found["volume_kernel"]) and {"values", "var_out"} <= set(found["softargmin_kernel"])
    assert {"p.corr", "p.out_corr", "p.D2"} <= set(found["geo_lookup_kernel"]) and "p.border" in found["warped_volume_kernel"]
    assert {"ad.align", "aw.scale"} <= set(found["upsample_softargmin_kernel"]) and "p.logits" in found["coex_regression_kernel"]
    assert {"ys", "coff"} <= set(found["ncdhw_to_ndhwc_kernel"])
    modes = set(selects)
    assert modes == set(NONCONV_MODE_VARIANTS), "modes without an entry in NONCONV_MODE_VARIANTS: %s; entries no field selects: %s" % (
        sorted(modes - set(NONCONV_MODE_VARIANTS)), sorted(set(NONCONV_MODE_VARIANTS) - modes))
    for mode, variants in NONCONV_MODE_VARIANTS.items():
        kernels = {v.split("<")[0] for v in variants}
        assert kernels == selects[mode], "mode %s lists instantiations of %s, but parameters of %s select it" % (
            mode, sorted(kernels), sorted(selects[mode]))
    plain = {r.fam for r in REGISTRY} - modes
    for mode, variants in NONCONV_MODE_VARIANTS.items():
        rows = [r for r in REGISTRY if r.fam == mode]
        assert rows, "mode %s has no row family" % mode
        assert mode not in plain
        got = {r.variant for r in rows}
        assert got == variants, "mode %s: instantiations without a row: %s; rows reaching an instantiation the mode does not: %s" % (
            mode, sorted(variants - got), sorted(got - variants))
    for fam in ("geov", "geomr"):
        rows = [r for r in REGISTRY if r.fam == fam]
        assert any(r.opts.get("cross") and r.opts["radius"] == 4 for r in rows), "%s: no row whose taps take the fallback read" % fam
        assert any(grid_z(r) == 65535 for r in rows), "%s: no row at grid z = 65535" % fam
    assert set(MODE_REQUIREMENTS) == set(NONCONV_MODE_VARIANTS)
    for mode, needs in MODE_REQUIREMENTS.items():
        rows = [r for r in REGISTRY if r.fam == mode]
        for what, met in needs.items():
            assert any(met(r) for r in rows), "mode %s: no row with %s" % (mode, what)
    for variant in ("warped_volume_kernel<8>", "warped_volume_kernel<16>"):      # CFNet's volume: (B, Cg, G, Cc, D, H, W)
        assert any(r.fam == "cas" and r.variant == variant and r.shape[1] > 0 and r.opts.get("mask") == 0 for r in REGISTRY), (
            "%s: no cas row with Cg > 0 and mask_left = 0" % variant)


def test_instance_norm_modes_have_contract_rows():
    """Every field of struct ConvParams is classified in CONV_PARAMS_FIELDS (tests/test_cuda_core_contract_gpu.py); the instance-norm
    rows reach every instantiation of the three _in_ entry points (dispatch_conv_k3's six, both transposed kernels, the 1x1 over one
    slab, two slabs and in 2D), each family has a row of more than 64 CTAs along grid x (not a multiple of 32) and a row with a large
    mean offset."""
    import re
    from test_cuda_core_contract_gpu import CONV_PARAMS_FIELDS, IN_FAMS, REGISTRY, in_grid
    fields = _struct_fields("conv3d.cu", "ConvParams")
    assert len(fields) == len(set(fields)) and {"in_stats", "ws_need", "vec_ok"} <= set(fields)
    assert set(fields) == set(CONV_PARAMS_FIELDS), "ConvParams fields not classified: %s; classified fields that are gone: %s" % (
        sorted(set(fields) - set(CONV_PARAMS_FIELDS)), sorted(set(CONV_PARAMS_FIELDS) - set(fields)))
    rows = [r for r in REGISTRY if r.fam in IN_FAMS]
    src = _csrc("conv3d.cu")
    dispatch = re.search(r"static int dispatch_conv_k3\(.*?\n\}", src, re.S).group(0)
    k3 = {"launch_conv_k3<%s>" % a.replace(" ", "") for a in re.findall(r"launch_conv_k3\s*<([^<>]*)>", dispatch)}
    assert len(k3) == 6 and {r.variant for r in rows if r.fam == "in-k3"} == k3
    assert {r.variant for r in rows if r.fam == "in-dc"} == {"launch_deconv<3,8>", "launch_deconv<4,8>"}
    pw = [r for r in rows if r.fam == "in-pw"]
    assert any(r.opts.get("c0", r.cin) < r.cin for r in pw) and any(r.opts.get("c0", r.cin) == r.cin and r.shape[1] > 1 for r in pw)
    assert any(r.shape[1] == 1 for r in pw)
    for fam in IN_FAMS:
        assert any(in_grid(r)[0] > 64 and in_grid(r)[0] % 32 for r in rows if r.fam == fam), "%s: no many-slot row" % fam
        assert any(r.opts.get("offset", 0) >= 20 for r in rows if r.fam == fam), "%s: no cancellation row" % fam
