"""GPU parity: rulebooks (bit-exact) and sparse convolutions (fp32, within 1e-4 relative -- the north-star bar)
against oracle/spconv_oracle.py, whose semantics are anchored on dense torch convs in tests/test_spconv_oracle.py."""
import numpy as np
import pytest
import torch

from oracle import spconv_oracle as so
from softgroup_b200 import spconv, synth
from softgroup_b200.configs import model_cfg
from softgroup_b200.model import SoftGroup

pytestmark = pytest.mark.gpu
# per-conv tolerance (relative to the output scale, vs the float64-accumulating oracle): the tensor-core path carries every
# operand as fp16 hi + fp16 lo and evaluates hi*hi + hi*lo + lo*hi with fp32 accumulation in wgmma (~2^-22 per product,
# 2^-25 absolute once lo is subnormal); the CUDA-core path is plain fp32 FFMA. Both far inside the 1e-4 end-to-end bar.
TOL = 5e-5


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.fixture(params=[0, 1], ids=['register_gather', 'smem_ring'])
def conv_kernel(request):
    """Every single-convolution parity case runs under both launches of the tensor-core kernel (spconv_tc.cu: one CTA per
    work item / persistent), named explicitly through sgb_spconv_forward_tc_ex, whatever sgb_spconv_kernel_choice would pick
    for the size."""
    from softgroup_b200.spconv import core
    old = core.CONV_KERNEL
    core.CONV_KERNEL = request.param
    yield request.param
    core.CONV_KERNEL = old


def _case(seed, shape=(23, 18, 15), B=2, C=8, density=0.2):
    rng = np.random.RandomState(seed)
    idx = []
    for b in range(B):
        occ = np.argwhere(rng.rand(*shape) < density)
        idx.append(np.concatenate([np.full((len(occ), 1), b), occ], 1))
    idx = np.concatenate(idx, 0).astype(np.int32)
    idx = idx[rng.permutation(len(idx))]
    return idx, rng.randn(len(idx), C).astype(np.float32), shape, B


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-12))


def test_rulebook_subm3_bitexact():
    idx, _, _, _ = _case(0)
    mp = spconv.build_subm_map(_cuda(idx)).cpu().numpy()
    assert np.array_equal(mp, so.subm_map(idx))


@pytest.mark.parametrize('shape', [(23, 18, 15), (16, 16, 16), (9, 33, 7)])
def test_rulebook_down2_bitexact(shape):
    idx, _, shape, _ = _case(1, shape=shape)
    out_idx, mp, inv, oshape = spconv.build_down_map(_cuda(idx), shape)
    o_idx, o_mp, o_inv, o_shape = so.down_map(idx, shape)
    assert oshape == o_shape
    assert np.array_equal(out_idx.cpu().numpy(), o_idx)
    assert np.array_equal(mp.cpu().numpy(), o_mp)
    assert np.array_equal(inv.cpu().numpy(), o_inv)


def test_rulebook_full_size():
    scan = synth.make_scan('c2_scannet', seed=0)
    import oracle
    vc, _, _ = oracle.voxelization_idx(scan['coords'], 1, 4)
    idx = vc.astype(np.int32)
    mp = spconv.build_subm_map(_cuda(idx)).cpu().numpy()
    assert np.array_equal(mp, so.subm_map(idx))
    out_idx, dmp, inv, _ = spconv.build_down_map(_cuda(idx), scan['spatial_shape'])
    o_idx, o_mp, o_inv, _ = so.down_map(idx, scan['spatial_shape'])
    assert np.array_equal(out_idx.cpu().numpy(), o_idx) and np.array_equal(dmp.cpu().numpy(), o_mp)
    assert np.array_equal(inv.cpu().numpy(), o_inv)


@pytest.mark.parametrize('Cin,Cout', [(6, 32), (32, 32), (64, 32), (96, 128), (16, 48), (224, 224)])
def test_subm_conv_vs_oracle(Cin, Cout, conv_kernel):
    idx, feats, _, _ = _case(Cin + Cout, C=Cin, density=0.25)
    rng = np.random.RandomState(2)
    W = (rng.randn(Cout, 3, 3, 3, Cin) / np.sqrt(27 * Cin)).astype(np.float32)
    conv = spconv.SubMConv3d(Cin, Cout, 3, padding=1, bias=False, indice_key='k').cuda()
    with torch.no_grad():
        conv.weight.copy_(torch.from_numpy(W))
        x = spconv.SparseConvTensor(_cuda(feats), _cuda(idx), (23, 18, 15), 2)
        y = conv(x)
    want = so.subm_conv3d(feats, idx, W, acc64=True)
    assert _rel(y.features.cpu().numpy(), want) < TOL
    assert 'k' in x.indice_dict


def _surface_case(seed, n_rows, extent=200):
    """Voxels on densely filled, gently warped plane patches (surface-like occupancy: ~9 of the 27 neighbours present,
    the statistics of a scanned room), enough rows to fill the machine with whole 128-row tiles."""
    rng = np.random.RandomState(seed)
    pts, have = [], 0
    while have < n_rows * 1.2:
        axis = rng.randint(3)
        c = rng.randint(10, extent - 10)
        w, h = rng.randint(50, 120, 2)
        u0, v0 = rng.randint(0, extent - w), rng.randint(0, extent - h)
        u, v = np.meshgrid(np.arange(u0, u0 + w), np.arange(v0, v0 + h), indexing='ij')
        u, v = u.ravel(), v.ravel()
        wob = np.round(np.sin(u / 9.0) * 2 + np.cos(v / 7.0) * 2).astype(np.int64)
        pts.append(np.insert(np.stack([u, v], 1), axis, c + wob, axis=1))
        have += len(u)
    idx = np.unique(np.concatenate(pts, 0), axis=0)
    idx = idx[rng.permutation(len(idx))][:n_rows]
    idx = np.concatenate([np.zeros((len(idx), 1), np.int64), idx], 1).astype(np.int32)
    return idx


def _rel_elem(got, want):
    """north star wording: float features within 1e-4 RELATIVE -- per element, with an absolute floor of 1e-6 of the
    tensor's largest magnitude for values that cancel to ~0: max over elements of |got-want| / (|want| + 1e-2 max|want|)
    would hide errors on small elements, so the bound is |got - want| <= tol * |want| + 1e-6 * max|want|."""
    floor = 1e-6 * np.abs(want).max()
    return float((np.maximum(np.abs(got - want) - floor, 0) / np.maximum(np.abs(want), 1e-30)).max())


@pytest.mark.parametrize('Cin,Cout,n_rows', [(32, 32, 40000), (64, 64, 24000), (96, 96, 24000), (128, 128, 20000),
                                             (192, 96, 20000), (64, 32, 40000), (224, 224, 20000)])
def test_subm_conv_bench_tile_configs_vs_oracle(Cin, Cout, n_rows, conv_kernel):
    """The tile configurations the 150k-point bench actually runs (>= 148 row tiles, more than the 132 SMs of an H100, so
    no column shrink / split-K of the small cases above): compared with the float64-accumulating oracle PER ELEMENT at the
    north-star tolerance."""
    idx = _surface_case(Cin * 7 + Cout, n_rows)
    rng = np.random.RandomState(Cin + Cout)
    feats = (rng.randn(len(idx), Cin) * rng.uniform(0.2, 3.0, size=(1, Cin))).astype(np.float32)
    W = (rng.randn(Cout, 3, 3, 3, Cin) / np.sqrt(12 * Cin)).astype(np.float32)
    scale, shift = rng.rand(Cin).astype(np.float32) + 0.5, rng.randn(Cin).astype(np.float32) * 0.3
    mp = so.subm_map(idx)
    assert (mp >= 0).sum(0).mean() > 5  # surface-like: several neighbours per row
    M = len(idx)
    assert M >= 148 * 128
    wk = torch.from_numpy(W.reshape(Cout, 27, Cin).transpose(1, 2, 0).copy()).cuda()
    out = spconv.conv_forward(_cuda(feats), Cin, 0, _cuda(mp), 27, M, wk, Cin, Cout, act=(_cuda(scale), _cuda(shift)))
    act = np.maximum(feats * scale + shift, 0).astype(np.float32)
    want = so.conv_from_map(act, mp, W, acc64=True)
    got = out.cpu().numpy()
    assert _rel(got, want) < TOL
    assert _rel_elem(got, want) < 1e-4


def test_conv_fused_act_residual_bias_strided(conv_kernel):
    idx, feats, _, _ = _case(5, C=40)
    rng = np.random.RandomState(3)
    M = len(idx)
    W = (rng.randn(24, 3, 3, 3, 40) / 30).astype(np.float32)
    scale, shift = rng.rand(40).astype(np.float32) + 0.5, rng.randn(40).astype(np.float32) * 0.3
    res = rng.randn(M, 24).astype(np.float32)
    bias = rng.randn(24).astype(np.float32)
    mp = so.subm_map(idx)
    wk = torch.from_numpy(W.reshape(24, 27, 40).transpose(1, 2, 0).copy()).cuda()
    out = torch.full((M, 64), 7.0, device='cuda')
    spconv.conv_forward(_cuda(feats), 40, 0, _cuda(mp), 27, M, wk, 40, 24, act=(_cuda(scale), _cuda(shift)),
                        residual=_cuda(res), bias=_cuda(bias), out=out, out_stride=64, out_off=32)
    act = np.maximum(feats * scale + shift, 0).astype(np.float32)
    want = so.conv_from_map(act, mp, W, acc64=True) + res + bias
    got = out.cpu().numpy()
    assert _rel(got[:, 32:56], want) < TOL
    assert np.all(got[:, :32] == 7.0) and np.all(got[:, 56:] == 7.0)


def test_down_and_inverse_modules(conv_kernel):
    idx, feats, shape, B = _case(7, C=32)
    rng = np.random.RandomState(4)
    Wd = (rng.randn(64, 2, 2, 2, 32) / 16).astype(np.float32)
    Wi = (rng.randn(32, 2, 2, 2, 64) / 8).astype(np.float32)
    down = spconv.SparseConv3d(32, 64, 2, stride=2, bias=False, indice_key='sp').cuda()
    inv = spconv.SparseInverseConv3d(64, 32, 2, bias=False, indice_key='sp').cuda()
    with torch.no_grad():
        down.weight.copy_(torch.from_numpy(Wd))
        inv.weight.copy_(torch.from_numpy(Wi))
        x = spconv.SparseConvTensor(_cuda(feats), _cuda(idx), shape, B)
        y = down(x)
        z = inv(y)
    o, o_idx, o_inv, o_shape = so.sparse_conv3d_k2s2(feats, idx, shape, Wd, acc64=True)
    assert np.array_equal(y.indices.cpu().numpy(), o_idx) and y.spatial_shape == o_shape
    assert _rel(y.features.cpu().numpy(), o) < TOL
    back = so.inverse_conv3d_k2(o, o_inv, Wi, acc64=True)
    assert np.array_equal(z.indices.cpu().numpy(), idx)
    assert _rel(z.features.cpu().numpy(), back) < TOL


def _randomize_bn(model, seed):
    g = torch.Generator().manual_seed(seed)
    for m in model.modules():
        if isinstance(m, torch.nn.BatchNorm1d):
            with torch.no_grad():
                m.running_mean.copy_(torch.randn(m.num_features, generator=g) * 0.1)
                m.running_var.copy_(torch.rand(m.num_features, generator=g) + 0.5)
                m.weight.copy_(torch.rand(m.num_features, generator=g) * 0.4 + 0.8)
                m.bias.copy_(torch.randn(m.num_features, generator=g) * 0.1)


@pytest.mark.parametrize('channels,num_blocks,shape,n', [(16, 4, 'c1_plumbing', 6000), (32, 7, 'c1_plumbing', 6000),
                                                         (32, 7, 'c2_scannet', 60000)])
def test_backbone_vs_oracle(channels, num_blocks, shape, n):
    """Whole sparse U-Net (53 SubM + 6 down + 6 inverse + 6 1x1 + 65 BN/ReLU at 32x7) vs the numpy restatement accumulating
    in float64 -- also at 60 000 points of the ScanNet-shape room (~58k voxels: levels 0-3 run the persistent ring kernel,
    the deep levels the split-K register-gather kernel, as in the bench)."""
    import oracle
    torch.manual_seed(0)
    scan = synth.make_scan(shape, seed=0, n_points=n)
    vc, v2p, p2v = oracle.voxelization_idx(scan['coords'], 1, 4)
    feats = np.concatenate([scan['feats'], scan['coords_float']], 1).astype(np.float32)
    vfeats = oracle.voxelization(feats, p2v, 4)
    model = SoftGroup(**model_cfg('scannet', channels=channels, num_blocks=num_blocks)).cuda().eval()
    _randomize_bn(model, 1)
    sd = {k: v.detach().cpu().numpy() for k, v in model.state_dict().items()}
    want = so.backbone(vfeats, vc.astype(np.int32), scan['spatial_shape'], sd, channels, num_blocks, acc64=True)
    with torch.no_grad():
        x = spconv.SparseConvTensor(_cuda(vfeats), _cuda(vc.astype(np.int32)), scan['spatial_shape'], 1)
        out = model.output_layer(model.unet(model.input_conv(x))).features.cpu().numpy()
    assert out.shape == want.shape
    assert _rel(out, want) < 1e-4  # north star: float features within 1e-4 relative
    np.testing.assert_allclose(out, want, rtol=1e-3, atol=1e-4 * np.abs(want).max())


@pytest.mark.parametrize('channels,num_blocks,n', [(16, 4, 6000), (32, 7, 30000)])
def test_plan_equals_module_path(channels, num_blocks, n):
    """The compiled launch plan (model/unet_plan.py, fused across modules) and the module path (fused inside each
    SparseSequential only, every block's input packed by act_pack) give bit-identical features, for the backbone (input
    conv + U-Net + output layer) and for the tiny U-Net of the instance branch (no input conv). The plan run one launch
    per call (use_plan = False) is bit-identical to its segmented run."""
    import oracle
    torch.manual_seed(0)
    scan = synth.make_scan('c2_scannet', seed=1, n_points=n)
    vc, v2p, p2v = oracle.voxelization_idx(scan['coords'], 1, 4)
    feats = np.concatenate([scan['feats'], scan['coords_float']], 1).astype(np.float32)
    vfeats = oracle.voxelization(feats, p2v, 4)
    model = SoftGroup(**model_cfg('scannet', channels=channels, num_blocks=num_blocks)).cuda().eval()
    _randomize_bn(model, 2)

    def run(use_plan, name, ic, un, ol, f, idx, shape, bs):
        model.use_plan = use_plan
        x = spconv.SparseConvTensor(f, idx, shape, bs)
        with torch.no_grad():
            return model._run_stack(name, ic, un, ol, x).clone()

    def modules(ic, un, ol, f, idx, shape, bs):
        x = spconv.SparseConvTensor(f, idx, shape, bs)
        with torch.no_grad():
            return ol(un(ic(x) if ic is not None else x)).features.clone()

    f, idx = _cuda(vfeats), _cuda(vc.astype(np.int32))
    a = run(True, 'backbone', model.input_conv, model.unet, model.output_layer, f, idx, scan['spatial_shape'], 1)
    b = modules(model.input_conv, model.unet, model.output_layer, f, idx, scan['spatial_shape'], 1)
    c = run(False, 'backbone', model.input_conv, model.unet, model.output_layer, f, idx, scan['spatial_shape'], 1)
    assert a.shape == b.shape and torch.equal(a, b)
    assert torch.equal(a, c)
    # tiny U-Net on a 20^3 grid per "proposal" (clusters_voxelization output shape)
    rng = np.random.RandomState(3)
    occ = np.argwhere(rng.rand(5, 20, 20, 20) < 0.08).astype(np.int32)
    tf = torch.from_numpy(rng.randn(len(occ), channels).astype(np.float32)).cuda()
    a = run(True, 'tiny', None, model.tiny_unet, model.tiny_unet_outputlayer, tf, _cuda(occ), [20, 20, 20], 5)
    b = modules(None, model.tiny_unet, model.tiny_unet_outputlayer, tf, _cuda(occ), [20, 20, 20], 5)
    c = run(False, 'tiny', None, model.tiny_unet, model.tiny_unet_outputlayer, tf, _cuda(occ), [20, 20, 20], 5)
    assert torch.equal(a, b)
    assert torch.equal(a, c)


def test_both_conv_kernels_bit_identical_and_choice():
    """The two launches evaluate the same products in the same order: bit-identical rows at a bench-size level
    (residual + bias + packed twin output), and sgb_spconv_kernel_choice follows the documented rule."""
    from softgroup_b200.ops import _lib
    from softgroup_b200.spconv import core
    L = _lib.lib()
    sms = torch.cuda.get_device_properties(0).multi_processor_count  # what the launch plans with (132 on H100 SXM5)
    assert L.sgb_spconv_kernel_choice(27, 137100, 32, 32, sms) == 1    # level 0: >= 4 * sms row tiles
    assert L.sgb_spconv_kernel_choice(27, 42391, 96, 96, sms) == 1     # level 2
    assert L.sgb_spconv_kernel_choice(27, 1933, 160, 160, sms) == 1    # level 4: 16 row tiles is the threshold
    assert L.sgb_spconv_kernel_choice(27, 1900, 160, 160, sms) == 0
    assert L.sgb_spconv_kernel_choice(27, 332, 192, 192, sms) == 0     # deep level: split-K clusters
    assert L.sgb_spconv_kernel_choice(27, 128 * (4 * sms - 1), 32, 32, sms) == 0  # 32-channel tiny U-Net: < 4 * sms tiles
    assert L.sgb_spconv_kernel_choice(27, 128 * 4 * sms, 32, 32, sms) == 1
    idx = _surface_case(11, 30000)
    rng = np.random.RandomState(5)
    Cin, Cout = 96, 64
    M = len(idx)
    feats = rng.randn(M, Cin).astype(np.float32)
    W = (rng.randn(Cout, 3, 3, 3, Cin) / np.sqrt(12 * Cin)).astype(np.float32)
    res, bias = rng.randn(M, Cout).astype(np.float32), rng.randn(Cout).astype(np.float32)
    mp = _cuda(so.subm_map(idx))
    wk = torch.from_numpy(W.reshape(Cout, 27, Cin).transpose(1, 2, 0).copy()).cuda()
    outs = []
    old = core.CONV_KERNEL
    try:
        for k in (0, 1):
            core.CONV_KERNEL = k
            emit = core.Emit(_cuda(rng.rand(Cout).astype(np.float32) * 0 + 1.5), _cuda(np.full(Cout, -0.25, np.float32)), key=None)
            y, pk = spconv.conv_forward(_cuda(feats), Cin, 0, mp, 27, M, wk, Cin, Cout, residual=_cuda(res), bias=_cuda(bias), emit=emit)
            outs.append((y.clone(), pk.clone()))
    finally:
        core.CONV_KERNEL = old
    assert torch.equal(outs[0][0], outs[1][0])
    assert torch.equal(outs[0][1].view(torch.int32), outs[1][1].view(torch.int32))


def test_activation_beyond_fp16_range_raises(conv_kernel):
    """|x| > 65504 cannot be carried by the fp16 hi/lo split: the packing code raises a flag and check_overflow() turns it
    into an exception (no silent saturation) -- from the input packer and from a producing conv's fused epilogue; the flag
    is cleared by the read, an in-range tensor afterwards passes."""
    from softgroup_b200.ops._lib import SgbError
    from softgroup_b200.spconv import core
    idx, feats, _, _ = _case(3, C=32)
    M = len(idx)
    mp = _cuda(so.subm_map(idx))
    rng = np.random.RandomState(0)
    wk = torch.from_numpy((rng.randn(27, 32, 32) / 30).astype(np.float32)).cuda()
    spconv.check_overflow()  # clean state
    big = feats.copy()
    big[5, 7] = 1.0e5
    spconv.conv_forward(_cuda(big), 32, 0, mp, 27, M, wk, 32, 32)  # the input packer sees the value
    with pytest.raises(SgbError):
        spconv.check_overflow()
    spconv.check_overflow()  # cleared
    # a producing conv whose consumer BatchNorm scales the output beyond the range: flagged by the fused epilogue
    emit = core.Emit(_cuda(np.full(32, 1.0e7, np.float32)), _cuda(np.zeros(32, np.float32)), key=None)
    spconv.conv_forward(_cuda(feats), 32, 0, mp, 27, M, wk, 32, 32, emit=emit)
    with pytest.raises(SgbError):
        spconv.check_overflow()
    spconv.conv_forward(_cuda(feats), 32, 0, mp, 27, M, wk, 32, 32)
    spconv.check_overflow()
