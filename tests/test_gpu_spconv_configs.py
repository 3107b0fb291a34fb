"""GPU parity of the sparse convolutions per element against the float64 oracle (oracle/spconv_oracle.py), for every tile
configuration the H100 runs (the case table of tests/spconv_cases.py, both launch forms of spconv_tc.cu), the packed
output contract (hi/lo fp16 rows, channel offsets, the fill of a half-written chunk, guard space), the whole backbone
of the 150k-point bench scan through the compiled plan, and the CUDA-core FFMA kernel (spconv.cu).

Two per-element bounds, with want the oracle and got the kernel:
  * the north-star bar  |got - want| <= 1e-4 |want| + 1e-6 max|want|;
  * a bound scaled by the magnitude of the sum, which stays tight where the sum cancels:
        |got - want| <= C_TC 2^-22 mag + 2^-24 |want|,
    mag = sum |a| |w| (the oracle on |act| and |W|, each floored at 2^-14 where non-zero: below the smallest normal fp16
    the lo half of the split keeps a fixed absolute precision) + |bias| + |residual|. The tensor-core path carries every
    operand as hi + lo 2^-11 and drops lo * lo: ~2^-22 per product."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import spconv_cases as sc  # noqa: E402
from oracle import spconv_oracle as so  # noqa: E402
from softgroup_b200 import spconv, synth  # noqa: E402
from softgroup_b200.configs import model_cfg  # noqa: E402
from softgroup_b200.model import SoftGroup  # noqa: E402
from softgroup_b200.ops import _lib  # noqa: E402
from softgroup_b200.ops._lib import check, ptr  # noqa: E402
from softgroup_b200.spconv import core  # noqa: E402

pytestmark = pytest.mark.gpu

# Measured on an H100 SXM5 over the case table: c <= 13.9 (tail_subm4, Cin 320, the longest accumulation chains without
# split-K; split-K ranks accumulate shorter chains and stay <= 2.1), packed rows <= 12.1 -- 16 leaves 15 % margin; the
# results are deterministic. Dropping the lo * hi product in spconv_tc_kernel<80> alone, or packing the weights with lo
# shift 10, fails every case that runs the changed code.
C_TC = 16.0
# CUDA-core fp32 (plain FFMA chains): |got - want| <= C_FFMA 2^-24 mag + 2^-24 |want|; measured <= 17.6 (K 27, Cin 600).
C_FFMA = 24.0
# With per-channel scales over 22 octaves, a few elements of a convolution cancel to ~1e-6 of their magnitude sum; there
# the tensor-core error (<= C_TC 2^-22 mag) exceeds 1e-4 |want| + 1e-6 max|want| (up to 0.29 relative at tail_subm4)
# while it is far inside the bound scaled by magnitude (the CUDA-core kernel meets the bar on the same inputs). The
# north-star bar is asserted on every element that keeps at least 2^-4 of its magnitude sum, where the bound above
# implies |got - want| <= 2^-14 |want| + 2^-24 |want| < 1e-4 |want|.
CANCELLED = 2.0**-4
FLOOR = 2.0**-14
SENT = np.int32(0x7FA5A5A5)  # a NaN pattern: guard words and columns must keep it


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _north_star(got, want, where=None):
    """max over elements (all, or those of `where`) of (|got - want| - 1e-6 max|want|) / |want| (<= 1e-4 is the bar)."""
    want = want.astype(np.float64)
    floor = 1e-6 * np.abs(want).max()
    r = np.maximum(np.abs(got - want) - floor, 0) / np.maximum(np.abs(want), 1e-30)
    return float(np.where(where, r, 0).max() if where is not None else r.max())


def _c_measured(got, want, mag, unit=2.0**-22):
    """Smallest c with |got - want| <= c unit mag + 2^-24 |want| for every element."""
    err = np.abs(got.astype(np.float64) - want) - 2.0**-24 * np.abs(want)
    assert np.all((mag > 0) | (err <= 0))
    return float((np.maximum(err, 0) / np.maximum(unit * mag, 1e-300)).max())


def _floored_abs(x):
    a = np.abs(x.astype(np.float64))
    return np.where(a > 0, np.maximum(a, FLOOR), 0)


def _features(rng, M, C):
    """Per-channel scales 2^-14 .. 2^8, exact zeros, and a BatchNorm whose shift makes a good share negative before the
    ReLU."""
    chs = 2.0**rng.uniform(-14, 8, size=C)
    x = rng.randn(M, C) * chs
    x[rng.rand(M, C) < 0.1] = 0
    scale = rng.uniform(0.5, 1.5, C)
    shift = rng.randn(C) * 0.5 * chs
    return x.astype(np.float32), scale.astype(np.float32), shift.astype(np.float32)


def _act64(x, scale, shift):
    return np.maximum(x.astype(np.float64) * scale.astype(np.float64) + shift.astype(np.float64), 0)


def _oracle(act, mp, W_kio):
    """float64-accumulated conv (conv_from_map) and its magnitude sum."""
    Wock = W_kio.transpose(2, 0, 1)
    want = so.conv_from_map(act, mp, Wock, acc64=True).astype(np.float64)
    mag = so.conv_from_map(_floored_abs(act), mp, _floored_abs(Wock), acc64=True).astype(np.float64)
    return want, mag


def _decode(pk_words, coff, C):
    """packed rows (float32-typed, [rows, stride words]) -> hi + lo 2^-11 of channels [coff, coff + C) in float64."""
    rows, stride = pk_words.shape
    h = pk_words.view(np.float16).reshape(rows, stride // 32, 2, 32).astype(np.float64)
    hi, lo = h[:, :, 0, :].reshape(rows, -1), h[:, :, 1, :].reshape(rows, -1)
    val = hi + lo * 2.0**-_lib.lib().sgb_spconv_lo_shift()
    return val[:, coff:coff + C]


def _half_bits(pk_words):
    """packed rows -> int16 [rows, chunks, 2 (hi, lo), 32 channels]."""
    rows, stride = pk_words.shape
    return pk_words.view(np.int16).reshape(rows, stride // 32, 2, 32)


def _channel_mask(stride, lo_ch, hi_ch):
    m = np.zeros(stride, bool)
    m[lo_ch:hi_ch] = True
    return np.broadcast_to(m.reshape(stride // 32, 1, 32), (stride // 32, 2, 32))


def _guarded(rows, cols):
    """[rows + 2, cols] int32 buffer of sentinels; the logical tensor is [1:-1]."""
    return torch.full((rows + 2, cols), int(SENT), dtype=torch.int32, device='cuda')


def _check_packed(buf, coff, Cout, fill, want, mag, ps, pb, tag):
    """buf: the guarded packed buffer (host int32) of relu(x ps + pb) for x = want (the conv). Channels
    [coff, coff + Cout) decode to it within ps (C_TC 2^-22 mag + 2^-24 |want|) (the conv's own bound through the
    BatchNorm) + 2^-22 |y| + 2^-34 (the fp32 fma and the hi/lo split); [coff + Cout, coff + N) are exactly zero; with
    fill, so is the rest of that 32-channel chunk; everything else keeps its sentinel. Returns the c needed."""
    N = (Cout + 15) // 16 * 16
    stride = buf.shape[1]
    words = buf.view(np.float32)
    sent_h = _half_bits(np.full((1, stride), SENT, np.int32).view(np.float32))[0]
    assert np.all(buf[0] == SENT) and np.all(buf[-1] == SENT), '%s: guard rows changed' % tag
    body = words[1:-1]
    hb = _half_bits(body)
    zero_hi = (coff + N + 31) // 32 * 32 if fill else coff + N
    written = _channel_mask(stride, coff, coff + Cout)
    zeros = _channel_mask(stride, coff + Cout, zero_hi)
    other = ~(written | _channel_mask(stride, coff + Cout, zero_hi))
    assert np.all(hb[:, zeros] == 0), '%s: padding / fill channels not zero' % tag
    assert np.all(hb[:, other] == sent_h[other]), '%s: a write outside the packed channels' % tag
    ref = np.maximum(want * ps + pb, 0)
    err = np.abs(_decode(body, coff, Cout) - ref) - (ps * 2.0**-24 * np.abs(want) + 2.0**-22 * np.abs(ref) + 2.0**-34)
    c = float((np.maximum(err, 0) / np.maximum(ps * 2.0**-22 * mag, 1e-300)).max())
    assert c <= C_TC, '%s: packed values need c = %g' % (tag, c)
    return c


# ---------------------------------------------------------------------------------------------------------------------
# the case table: rulebooks of the bench scan, random rulebooks for the synthetic cases
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def bench_levels():
    """Indices and rulebooks of every U-Net level of the bench scan (seed 0, 150k points), from the oracle."""
    import oracle
    scan = synth.make_scan('c2_scannet', seed=sc.BENCH_SEED, n_points=sc.BENCH_POINTS)
    vc, _, _ = oracle.voxelization_idx(scan['coords'], 1, 4)
    idx, shape = vc.astype(np.int32), scan['spatial_shape']
    levels = []
    for i in range(len(sc.BENCH_ROWS)):
        lv = dict(idx=idx, subm=so.subm_map(idx))
        if i + 1 < len(sc.BENCH_ROWS):
            idx, lv['down'], lv['inv'], shape = so.down_map(idx, shape)
        levels.append(lv)
    assert tuple(len(lv['idx']) for lv in levels) == sc.BENCH_ROWS
    return levels


def _rand_map(rng, K, Mout, Min):
    """Random rulebook: ~40 % of the pairs present, two offsets absent everywhere, and the rows of one 128-row tile
    (the middle one, or all of them below two tiles) without any neighbour -- skipped offsets and empty tiles."""
    mp = np.where(rng.rand(K, Mout) < 0.4, rng.randint(0, Min, size=(K, Mout)), -1).astype(np.int32)
    if K > 2:
        mp[rng.choice(K, 2, replace=False)] = -1
    t = (Mout // 128) // 2
    mp[:, t * 128:(t + 1) * 128] = -1
    return mp


def _case_map(case, levels):
    if case.kind == 'ident':
        return None
    if case.kind == 'rand':
        return _rand_map(np.random.RandomState(len(case.name) * 7 + case.Cin), case.K, case.Mout, case.Min)
    lv = levels[case.level]
    return lv[case.kind]


@pytest.mark.parametrize('case', sc.CASES, ids=[c.name for c in sc.CASES])
def test_conv_case_vs_oracle(case, bench_levels):
    """One convolution of the table under both launch forms (named explicitly): input BatchNorm+ReLU, bias, residual,
    strided fp32 output with guard columns / rows, and the packed output of a consumer BatchNorm+ReLU; the two forms
    are bit-identical wherever the one-CTA-per-item launch has no split-K."""
    L = _lib.lib()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.RandomState(sc.CASES.index(case) + 100)
    mp = _case_map(case, bench_levels)
    assert mp is None or mp.shape == (case.K, case.Mout)
    K, Mout, Min, Cin, Cout = case.K, case.Mout, case.Min, case.Cin, case.Cout
    x, s_in, b_in = _features(rng, Min, Cin)
    W = (rng.randn(K, Cin, Cout) / np.sqrt(9 * Cin)).astype(np.float32)
    W[rng.rand(K, Cin, Cout) < 0.02] = 0
    act = _act64(x, s_in, b_in)
    conv, mag = _oracle(act, mp if mp is not None else np.arange(Mout, dtype=np.int32)[None], W)
    osc = np.abs(conv).max() + 1e-30
    bias = (rng.randn(Cout) * 0.1 * osc).astype(np.float32)
    res = (rng.randn(Mout, Cout) * 0.5 * osc).astype(np.float32)
    want = conv + bias + res
    mag = mag + np.abs(bias) + np.abs(res)
    ps = rng.uniform(0.5, 1.5, Cout).astype(np.float32)
    pb = (rng.randn(Cout) * 0.3 * np.abs(want).mean(0)).astype(np.float32)

    out_off, out_stride = 3, Cout + 8
    pk_stride = (Cout + 31) // 32 * 32 + 32  # one guard chunk per row
    d_x, d_mp, d_W = _cuda(x), (_cuda(mp) if mp is not None else None), core.WeightPack(_cuda(W))
    runs = {}
    old = core.CONV_KERNEL
    try:
        for form in (0, 1):
            core.CONV_KERNEL = form
            out = torch.full((Mout + 2, out_stride), float('nan'), device='cuda')
            out.view(torch.int32).fill_(int(SENT))
            pk = _guarded(Mout, pk_stride)
            emit = core.Emit(_cuda(ps), _cuda(pb), key=None, buf=pk[1:-1].view(torch.float32), coff=0, fill=True)
            spconv.conv_forward(d_x, Cin, 0, d_mp, K, Mout, d_W, Cin, Cout, act=(_cuda(s_in), _cuda(b_in)), bias=_cuda(bias),
                                residual=_cuda(res), out=out[1:-1], out_stride=out_stride, out_off=out_off, emit=emit, m_in=Min)
            spconv.check_overflow()
            runs[form] = (out.cpu().numpy(), pk.cpu().numpy())
    finally:
        core.CONV_KERNEL = old
    kept = np.abs(want) >= CANCELLED * mag
    for form, (out, pk) in runs.items():
        a = sc.launch(case, form, sms, L)
        tag = '%s form %d (NT %d x %d, S %d)' % (case.name, form, a['NT'], a['parts'], a['S'])
        ob = out.view(np.int32)
        assert np.all(ob[0] == SENT) and np.all(ob[-1] == SENT), tag + ': guard rows of the fp32 output changed'
        assert np.all(ob[1:-1, :out_off] == SENT) and np.all(ob[1:-1, out_off + Cout:] == SENT), tag + ': guard columns'
        got = out[1:-1, out_off:out_off + Cout]
        c = _c_measured(got, want, mag)
        c_pk = _check_packed(pk, 0, Cout, True, want, mag, ps.astype(np.float64), pb.astype(np.float64), tag)
        ns_all, ns = _north_star(got, want), _north_star(got, want, kept)
        print('\n[spconv case] %-18s form %d NT %3d x %d S %d: c %.3f, packed c %.3f, north-star %.3e (all elements %.3e, '
              '%d cancelled below %g of their magnitude)' % (case.name, form, a['NT'], a['parts'], a['S'], c, c_pk, ns, ns_all,
                                                              (~kept).sum(), CANCELLED))
        assert c <= C_TC, '%s: c = %.3f' % (tag, c)
        assert ns <= 1e-4, '%s: north-star %.3e' % (tag, ns)
    if sc.launch(case, 0, sms, L)['S'] == 1:
        assert np.array_equal(runs[0][0].view(np.int32), runs[1][0].view(np.int32)), case.name + ': fp32 rows differ'
        assert np.array_equal(runs[0][1], runs[1][1]), case.name + ': packed rows differ'


# ---------------------------------------------------------------------------------------------------------------------
# packed-output contract at the C ABI: channel offsets, fill, guard space
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('kernel', [0, 1])
@pytest.mark.parametrize('fill', [0, 1])
@pytest.mark.parametrize('Cout', [13, 16, 32])
@pytest.mark.parametrize('coff', [0, 8, 16, 24, 32])
def test_forward_tc_packed_output_contract(coff, Cout, fill, kernel):
    """sgb_spconv_forward_tc_ex writing packed rows at channel offset `coff` (N % 32 = 16 and 0, padding channels at
    Cout = 13) into a buffer of sentinel guard rows and columns: values, exact zeros, the fill of the chunk the written
    channels end in, and no write anywhere else -- in particular not below coff and not past the fill."""
    L = _lib.lib()
    rng = np.random.RandomState(coff * 7 + Cout + 100 * fill)
    K, Mout, Min, Cin = 8, 300, 500, 40
    x = rng.randn(Min, Cin).astype(np.float32)
    W = (rng.randn(K, Cin, Cout) / 12).astype(np.float32)
    mp = _rand_map(rng, K, Mout, Min)
    ps, pb = rng.uniform(0.5, 1.5, Cout).astype(np.float32), rng.randn(Cout).astype(np.float32) * 0.3
    want, mag = _oracle(x, mp, W)
    pk_in = core.act_pack(_cuda(x), Cin, 0, Cin)
    N = (Cout + 15) // 16 * 16
    stride = (coff + N + 31) // 32 * 32 + 32
    buf = _guarded(Mout, stride)
    Wp = core.pack_weight_tc(_cuda(W))
    d_mp, d_ps, d_pb = _cuda(mp), _cuda(ps), _cuda(pb)
    check(L.sgb_spconv_forward_tc_ex(ptr(pk_in), pk_in.size(1), Min, ptr(d_mp), K, Mout, ptr(Wp), Cin, Cout, None, 0, 0, None,
                                     None, 0, 0, ptr(buf[1:-1]), stride, coff, ptr(d_ps), ptr(d_pb), 1, fill, kernel,
                                     core._stream()), 'sgb_spconv_forward_tc_ex')
    _check_packed(buf.cpu().numpy(), coff, Cout, fill, want, mag, ps.astype(np.float64), pb.astype(np.float64),
                  'coff %d Cout %d fill %d kernel %d' % (coff, Cout, fill, kernel))


@pytest.mark.parametrize('C,wide', [(13, False), (13, True), (16, False), (16, True), (32, False), (40, True)])
@pytest.mark.parametrize('coff', [0, 8, 16, 24, 32])
def test_act_pack_contract(coff, C, wide):
    """sgb_act_pack at channel offset `coff` of a guarded buffer: C channels of relu(x scale + shift), zeros up to Cfill
    (C rounded up to even, or -- `wide` -- up to the end of the 32-channel chunk), sentinels everywhere else."""
    L = _lib.lib()
    rng = np.random.RandomState(coff + C)
    M, x_off, x_stride = 257, 5, C + 9
    x = (rng.randn(M, x_stride) * 2.0**rng.uniform(-14, 8, size=x_stride)).astype(np.float32)
    s, b = rng.uniform(0.5, 1.5, C).astype(np.float32), (rng.randn(C) * 0.1).astype(np.float32)
    Cfill = (coff + C + 31) // 32 * 32 - coff if wide else (C + 1) // 2 * 2
    stride = (coff + Cfill + 31) // 32 * 32 + 32
    buf = _guarded(M, stride)
    d_x, d_s, d_b = _cuda(x), _cuda(s), _cuda(b)  # alive until the kernel has read them
    check(L.sgb_act_pack(ptr(d_x), x_stride, x_off, ptr(d_s), ptr(d_b), 1, ptr(buf[1:-1]), stride, coff, M, C, Cfill,
                         core._stream()), 'sgb_act_pack')
    want = _act64(x[:, x_off:x_off + C], s, b)
    got = buf.cpu().numpy()
    # the fill region of _check_packed is [coff + C, round_up32(coff + N)): express Cfill through (Cout, fill)
    h = got.view(np.float32)
    hb = _half_bits(h[1:-1])
    sent_h = _half_bits(np.full((1, stride), SENT, np.int32).view(np.float32))[0]
    assert np.all(got[0] == SENT) and np.all(got[-1] == SENT)
    zeros = _channel_mask(stride, coff + C, coff + Cfill)
    other = ~_channel_mask(stride, coff, coff + Cfill)
    assert np.all(hb[:, zeros] == 0) and np.all(hb[:, other] == sent_h[other])
    err = np.abs(_decode(h[1:-1], coff, C) - want)
    assert np.all(err <= 2.0**-22 * np.abs(want) + 2.0**-34)


# ---------------------------------------------------------------------------------------------------------------------
# whole networks through the compiled plan
# ---------------------------------------------------------------------------------------------------------------------
def _randomize_bn(model, seed):
    g = torch.Generator().manual_seed(seed)
    for m in model.modules():
        if isinstance(m, torch.nn.BatchNorm1d):
            with torch.no_grad():
                m.running_mean.copy_(torch.randn(m.num_features, generator=g) * 0.1)
                m.running_var.copy_(torch.rand(m.num_features, generator=g) + 0.5)
                m.weight.copy_(torch.rand(m.num_features, generator=g) * 0.4 + 0.8)
                m.bias.copy_(torch.randn(m.num_features, generator=g) * 0.1)


def test_backbone_bench_scan_plan_vs_oracle():
    """The backbone of the bench workload exactly as bench.py runs it (seed-0 c2_scannet scan at 150k points, scannet
    config 32 x 7, the compiled plan) against the float64 oracle, per element at the north-star bar."""
    import oracle
    torch.manual_seed(0)
    scan = synth.make_scan('c2_scannet', seed=sc.BENCH_SEED, n_points=sc.BENCH_POINTS)
    vc, _, p2v = oracle.voxelization_idx(scan['coords'], 1, 4)
    feats = np.concatenate([scan['feats'], scan['coords_float']], 1).astype(np.float32)
    vfeats = oracle.voxelization(feats, p2v, 4)
    model = SoftGroup(**model_cfg('scannet')).cuda().eval()
    _randomize_bn(model, 1)
    model.use_plan = True
    sd = {k: v.detach().cpu().numpy() for k, v in model.state_dict().items()}
    want = so.backbone(vfeats, vc.astype(np.int32), scan['spatial_shape'], sd, 32, 7, acc64=True)
    with torch.no_grad():
        x = spconv.SparseConvTensor(_cuda(vfeats), _cuda(vc.astype(np.int32)), scan['spatial_shape'], 1)
        got = model._run_stack('backbone', model.input_conv, model.unet, model.output_layer, x).cpu().numpy()
    spconv.check_overflow()
    assert len(model._plans) == 1 and got.shape == want.shape == (sc.BENCH_ROWS[0], 32)
    ns = _north_star(got, want)
    print('\n[backbone 150k plan] per-element north-star %.3e, max |err| / max |want| %.3e' %
          (ns, np.abs(got - want).max() / np.abs(want).max()))
    assert ns <= 1e-4


def test_tiny_unet_plan_vs_oracle():
    """The instance branch's tiny U-Net ([32, 64]) through the compiled plan on a batch of 64 proposal grids (20^3,
    clusters of surface-like voxels), against so.ublock + the output BatchNorm+ReLU in float64."""
    torch.manual_seed(0)
    model = SoftGroup(**model_cfg('scannet')).cuda().eval()
    _randomize_bn(model, 3)
    model.use_plan = True
    rng = np.random.RandomState(4)
    occ = []
    for b in range(64):  # a shell of an ellipsoid per proposal: a scanned object's surface
        c, r = rng.uniform(7, 13, 3), rng.uniform(3, 9, 3)
        g = np.argwhere(np.ones((20, 20, 20), bool))
        d = np.sqrt((((g - c) / r)**2).sum(1))
        g = g[(np.abs(d - 1) < 0.18) | ((rng.rand(len(g)) < 0.01) & (d < 1))]
        occ.append(np.concatenate([np.full((len(g), 1), b), g], 1))
    idx = np.concatenate(occ, 0).astype(np.int32)
    idx = idx[rng.permutation(len(idx))]
    f = (rng.randn(len(idx), 32) * rng.uniform(0.2, 3, size=32)).astype(np.float32)
    sd = {k: v.detach().cpu().numpy() for k, v in model.state_dict().items()}
    want = so.ublock(f, idx, [20, 20, 20], sd, 'tiny_unet', [32, 64], acc64=True)
    want = so._bn_relu(want, sd, 'tiny_unet_outputlayer.0', acc64=True)
    with torch.no_grad():
        x = spconv.SparseConvTensor(_cuda(f), _cuda(idx), [20, 20, 20], 64)
        got = model._run_stack('tiny', None, model.tiny_unet, model.tiny_unet_outputlayer, x).cpu().numpy()
    assert 'tiny' in model._plans and got.shape == want.shape
    ns = _north_star(got, want)
    print('\n[tiny U-Net plan] %d rows: per-element north-star %.3e' % (len(idx), ns))
    assert ns <= 1e-4


# ---------------------------------------------------------------------------------------------------------------------
# the CUDA-core FFMA kernel (Cin > 512 or Cout > 256, and SGB_CONV_IMPL=ffma)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('Cout', [24, 300])
@pytest.mark.parametrize('Cin', [6, 40, 600])
@pytest.mark.parametrize('K', [1, 8, 27])
def test_ffma_conv_vs_oracle(K, Cin, Cout):
    """sgb_spconv_forward per element against the float64 oracle: scalar gather (in_off not a multiple of 4) and float4
    gather, with and without the fused input BatchNorm+ReLU, residual at res_off, bias, strided output with sentinels."""
    L = _lib.lib()
    rng = np.random.RandomState(K * 1000 + Cin + Cout)
    Mout, Min = 700, 900
    mp = _rand_map(rng, K, Mout, Min) if K > 1 else None
    W = (rng.randn(K, Cin, Cout) / np.sqrt(9 * Cin)).astype(np.float32)
    bias = rng.randn(Cout).astype(np.float32)
    res_off, res_stride = 2, Cout + 5
    res = rng.randn(Mout, res_stride).astype(np.float32)
    for in_off, use_act in ((3, True), (4, False), (4, True), (3, False)):
        in_stride = in_off + Cin + (4 - (in_off + Cin) % 4) % 4  # multiple of 4: the float4 path is up to in_off
        x = np.zeros((Min, in_stride), np.float32)
        xs, s, b = _features(rng, Min, Cin)
        x[:, in_off:in_off + Cin] = xs
        act = _act64(xs, s, b) if use_act else xs.astype(np.float64)
        conv, mag = _oracle(act, mp if mp is not None else np.arange(Mout, dtype=np.int32)[None], W)
        want = conv + bias + res[:, res_off:res_off + Cout]
        mag = mag + np.abs(bias) + np.abs(res[:, res_off:res_off + Cout])
        out_off, out_stride = 1, Cout + 3
        out = torch.full((Mout + 2, out_stride), 0, dtype=torch.int32, device='cuda').fill_(int(SENT))
        d_s, d_b = (_cuda(s), _cuda(b)) if use_act else (None, None)
        d_mp = _cuda(mp) if mp is not None else None
        d_x, d_W, d_res, d_bias = _cuda(x), _cuda(W), _cuda(res), _cuda(bias)  # alive until the kernel has read them
        check(L.sgb_spconv_forward(ptr(d_x), in_stride, in_off, ptr(d_mp), K, Mout, ptr(d_W), Cin, Cout, ptr(d_s), ptr(d_b),
                                   ptr(d_res), res_stride, res_off, ptr(d_bias), ptr(out[1:-1]), out_stride, out_off,
                                   core._stream()), 'sgb_spconv_forward')
        ob = out.cpu().numpy()
        assert np.all(ob[0] == SENT) and np.all(ob[-1] == SENT)
        assert np.all(ob[1:-1, :out_off] == SENT) and np.all(ob[1:-1, out_off + Cout:] == SENT)
        got = ob[1:-1, out_off:out_off + Cout].view(np.float32)
        ns, c = _north_star(got, want), _c_measured(got, want, mag, unit=2.0**-24)
        print('\n[ffma] K %d Cin %d Cout %d in_off %d act %d: north-star %.3e, c %.3f' % (K, Cin, Cout, in_off, use_act, ns, c))
        assert ns <= 1e-4 and c <= C_FFMA


def test_conv_forward_sends_wide_outputs_to_ffma(monkeypatch):
    """Under the default tensor-core setting, Cout > 256 runs the CUDA-core kernel (and its result is the oracle's);
    Cout <= 256 runs the tensor-core kernel."""
    assert core.CONV_IMPL == 'tc'
    real, called = _lib.lib(), []

    class Spy(object):
        def __getattr__(self, name):
            if name.startswith('sgb_spconv_forward'):
                called.append(name)
            return getattr(real, name)

    monkeypatch.setattr(_lib, 'lib', lambda: Spy())
    rng = np.random.RandomState(9)
    M, Cin = 500, 64
    mp = _rand_map(rng, 27, M, M)
    x = rng.randn(M, Cin).astype(np.float32)
    for Cout, name in ((300, 'sgb_spconv_forward'), (256, 'sgb_spconv_forward_tc_ex')):
        W = (rng.randn(27, Cin, Cout) / 20).astype(np.float32)
        called.clear()
        got = spconv.conv_forward(_cuda(x), Cin, 0, _cuda(mp), 27, M, _cuda(W), Cin, Cout).cpu().numpy()
        assert called == [name]
        want, mag = _oracle(x, mp, W)
        assert _north_star(got, want) <= 1e-4


def test_backbone_ffma_module_path_vs_oracle():
    """The whole backbone at 60k points with SGB_CONV_IMPL=ffma: the unfused SparseSequential path (BatchNorm flushes,
    act= fused into the FFMA gather, no plan) against the float64 oracle per element."""
    import oracle
    torch.manual_seed(0)
    scan = synth.make_scan('c2_scannet', seed=0, n_points=60000)
    vc, _, p2v = oracle.voxelization_idx(scan['coords'], 1, 4)
    feats = np.concatenate([scan['feats'], scan['coords_float']], 1).astype(np.float32)
    vfeats = oracle.voxelization(feats, p2v, 4)
    model = SoftGroup(**model_cfg('scannet')).cuda().eval()
    _randomize_bn(model, 1)
    model.use_plan = True  # ignored under ffma: _run_stack takes the module path
    sd = {k: v.detach().cpu().numpy() for k, v in model.state_dict().items()}
    want = so.backbone(vfeats, vc.astype(np.int32), scan['spatial_shape'], sd, 32, 7, acc64=True)
    old = core.CONV_IMPL
    core.CONV_IMPL = 'ffma'
    try:
        with torch.no_grad():
            x = spconv.SparseConvTensor(_cuda(vfeats), _cuda(vc.astype(np.int32)), scan['spatial_shape'], 1)
            got = model._run_stack('backbone', model.input_conv, model.unet, model.output_layer, x).cpu().numpy()
    finally:
        core.CONV_IMPL = old
    assert not model._plans
    ns = _north_star(got, want)
    print('\n[backbone 60k ffma] per-element north-star %.3e' % ns)
    assert ns <= 1e-4
