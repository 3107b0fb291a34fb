"""spconv-shaped surface used by the reference model, on libsgb200 kernels (no spconv dependency).

Covers exactly what softgroup/model/blocks.py, softgroup/model/softgroup.py and softgroup/util/fp16.py touch
(SURVEY.md 8b): SparseConvTensor(.features .indices .spatial_shape .batch_size .indice_dict .grid
.replace_feature), SparseSequential, SparseModule, SubMConv3d / SparseConv3d / SparseInverseConv3d with
`.weight [out,k,k,k,in]`, `.in_channels`, `.out_channels`, `.bias`, `indice_key` rulebook sharing.

Inference-only: BatchNorm1d must be in eval mode; it is folded to (scale, shift) and, together with a following
ReLU, fused into the input transform of the next sparse convolution (the pre-activation pattern of
blocks.py:55-70). SparseSequential does that peephole fusion itself, so the reference's module tree and
state_dict names stay untouched.
"""
import ctypes
import os
import weakref
from collections import OrderedDict

import torch
from torch import nn

from .. import profiler
from ..ops import _lib
from ..ops._lib import check, ptr, stream as _stream, workspace as _ws


class SparseConvTensor(object):

    def __init__(self, features, indices, spatial_shape, batch_size, grid=None, indice_dict=None):
        self.features = features
        self.indices = indices
        self.spatial_shape = [int(s) for s in spatial_shape]
        self.batch_size = batch_size
        self.indice_dict = indice_dict if indice_dict is not None else {}
        self.grid = grid

    def replace_feature(self, feature):
        out = SparseConvTensor(feature, self.indices, self.spatial_shape, self.batch_size, self.grid,
                               self.indice_dict)
        return out

    @property
    def spatial_size(self):
        n = 1
        for s in self.spatial_shape:
            n *= s
        return n

    def find_indice_pair(self, key):
        if key is None:
            return None
        return self.indice_dict.get(key, None)


class SparseModule(nn.Module):
    """Marker base class (spconv.pytorch.modules.SparseModule; blocks.py:5,44)."""
    pass


# ---------------------------------------------------------------------------------------------------------
# BatchNorm folding (eval mode), cached per module and invalidated when any parameter/buffer changes
# ---------------------------------------------------------------------------------------------------------
_bn_cache = weakref.WeakKeyDictionary()


def fold_bn(bn):
    """-> (scale, shift) float32 CUDA tensors with y = x*scale + shift == BatchNorm1d(eval)(x)."""
    if bn.training:
        raise RuntimeError('softgroup_b200 sparse modules are inference-only: call model.eval() '
                           '(BatchNorm1d in training mode cannot be folded)')
    ver = (bn.weight._version, bn.bias._version, bn.running_mean._version, bn.running_var._version,
           bn.weight.data_ptr(), bn.running_mean.data_ptr())
    hit = _bn_cache.get(bn)
    if hit is not None and hit[0] == ver:
        return hit[1], hit[2]
    with torch.no_grad():
        inv = torch.rsqrt(bn.running_var.double() + bn.eps)
        scale = bn.weight.double() * inv
        shift = bn.bias.double() - bn.running_mean.double() * scale
        scale, shift = scale.float().contiguous(), shift.float().contiguous()
    _bn_cache[bn] = (ver, scale, shift)
    return scale, shift


def bn_relu_rows(x, scale, shift, relu):
    """Standalone BatchNorm(eval)(+ReLU) over the rows of a dense [M,C] tensor."""
    x = x.contiguous()
    y = torch.empty_like(x)
    M, C = x.shape
    with profiler.record('bn_relu', 8 * M * C):
        check(_lib.lib().sgb_bn_relu(ptr(x), C, ptr(scale), ptr(shift), int(relu), ptr(y), C, M, C, _stream()),
              'sgb_bn_relu')
    return y


# ---------------------------------------------------------------------------------------------------------
# rulebooks
# ---------------------------------------------------------------------------------------------------------
def _indices_i32(indices):
    if indices.dtype != torch.int32:
        indices = indices.int()
    return indices.contiguous()


def build_subm_map(indices):
    L = _lib.lib()
    indices = _indices_i32(indices)
    M = indices.size(0)
    mp = torch.empty((27, M), dtype=torch.int32, device=indices.device)
    ws = _ws(L.sgb_rulebook_workspace_bytes(M), indices.device)
    with profiler.record('rulebook_subm3', 16 * M + 4 * 27 * M):
        check(L.sgb_rulebook_subm3(ptr(indices), M, ptr(mp), ptr(ws), ws.numel(), _stream()), 'sgb_rulebook_subm3')
    return mp


def build_down_map(indices, spatial_shape):
    L = _lib.lib()
    indices = _indices_i32(indices)
    M = indices.size(0)
    dev = indices.device
    ws = _ws(L.sgb_rulebook_workspace_bytes(M), dev)
    shp = (ctypes.c_int * 3)(*[int(s) for s in spatial_shape])
    with profiler.record('rulebook_down2', 16 * M + 4 * 9 * M):
        Mout = check(L.sgb_rulebook_down2_count(ptr(indices), M, shp, ptr(ws), ws.numel(), _stream()),
                     'sgb_rulebook_down2_count')
    out_indices = torch.empty((Mout, 4), dtype=torch.int32, device=dev)
    mp = torch.empty((8, Mout), dtype=torch.int32, device=dev)
    inv = torch.empty((8, M), dtype=torch.int32, device=dev)
    check(
        L.sgb_rulebook_down2_fill(ptr(indices), M, Mout, ptr(out_indices), ptr(mp), ptr(inv), ptr(ws), ws.numel(),
                                  _stream()), 'sgb_rulebook_down2_fill')
    return out_indices, mp, inv, [int(s) // 2 for s in spatial_shape]


def rulebook(indice_dict, key, kind, indices, spatial_shape=None):
    """The rulebook of indice_key `key` over the sites `indices`, built on first use and shared through `indice_dict`.
    kind 'subm': {'map'}; kind 'down' (k2 s2, and its inverse): {'map', 'inv_map', 'out_indices', 'out_shape',
    'in_indices', 'in_shape'}."""
    rb = indice_dict.get(key) if key is not None else None
    if rb is None:
        if kind == 'subm':
            rb = {'kind': 'subm', 'map': build_subm_map(indices)}
        else:
            out_indices, mp, inv, out_shape = build_down_map(indices, spatial_shape)
            rb = {'kind': 'down', 'map': mp, 'inv_map': inv, 'out_indices': out_indices, 'out_shape': out_shape,
                  'in_indices': indices, 'in_shape': spatial_shape}
        if key is not None:
            indice_dict[key] = rb
    return rb


CONV_IMPL = os.environ.get('SGB_CONV_IMPL', 'tc')  # 'tc' = wgmma tensor cores (default), 'ffma' = CUDA-core fp32 (A/B only)
# which of the two launches of the tensor-core kernel the module path asks for: -1 = the library chooses (sgb_spconv_kernel_choice), 0 = register
# gather, 1 = persistent shared-memory ring. Parity tests run every case under 0 and 1; the compiled plan always uses -1.
CONV_KERNEL = -1


def pack_weight_tc(W):
    """[K, Cin, Cout] f32 -> packed fp16 split for sgb_spconv_forward_tc (layout in sgb200.h):
    [K, nkc, 4 chunks, 2 (hi, lo), N, 8 halves], hi = fp16(W), lo = fp16((W - hi) * 2^sgb_spconv_lo_shift());
    returned as a float32-typed buffer."""
    K, Cin, Cout = W.shape
    N = (Cout + 15) // 16 * 16
    nkc = (Cin + 31) // 32
    Wp = torch.zeros((K, nkc * 32, N), dtype=torch.float32, device=W.device)
    Wp[:, :Cin, :Cout] = W
    Wp = Wp.view(K, nkc, 4, 8, N).permute(0, 1, 2, 4, 3).contiguous()  # [K, nkc, 4, N, 8]
    hi = Wp.half()
    lo = ((Wp - hi.float()) * float(2 ** _lib.lib().sgb_spconv_lo_shift())).half()  # same scaling as the kernel
    packed = torch.stack([hi, lo], dim=3).contiguous()  # [K, nkc, 4, 2, N, 8] fp16
    return packed.view(torch.float32)


class WeightPack(object):
    """Weight of one conv in the kernels' formats: .kio [K,Cin,Cout] (CUDA-core kernel) and .tc(), the packed fp16
    hi/lo split of the tensor-core kernel."""
    __slots__ = ('kio', 'packed')

    def __init__(self, kio):
        self.kio = kio
        self.packed = None

    def tc(self):
        if self.packed is None:
            self.packed = pack_weight_tc(self.kio)
        return self.packed


def pack_fill(C, width, coff):
    """Channels sgb_act_pack writes when it packs C channels at channel `coff` of a packed buffer `width` channels wide:
    C when they end on a 32-channel boundary, else C rounded up to 32, the rest zeroed (never past `width`)."""
    return min(width - coff, (C + 31) // 32 * 32) if (coff + C) % 32 else C


def act_pack(feats, in_stride, in_off, C, act=None, relu=None, out=None, out_coff=0, rows=None):
    """fp32 rows -> packed rows (per 32-channel chunk: 16 words fp16 hi pairs | 16 words lo pairs) after the optional
    BatchNorm(eval) `act = (scale, shift)` and ReLU. `out`: an existing packed buffer [M, cpad] float32-typed (concat
    halves); returns the packed buffer."""
    M = feats.size(0) if rows is None else rows
    if relu is None:
        relu = act is not None
    if out is None:
        out = torch.empty((M, (C + 31) // 32 * 32), dtype=torch.float32, device=feats.device)
    cpad = out.size(1)
    fill = pack_fill(C, cpad, out_coff)
    scale, shift = act if act is not None else (None, None)
    with profiler.record('act_pack', 8 * M * C):
        check(_lib.lib().sgb_act_pack(ptr(feats), in_stride, in_off, ptr(scale), ptr(shift), int(bool(relu)), ptr(out),
                                      cpad, out_coff, M, C, fill, _stream()), 'sgb_act_pack')
    return out


def check_overflow():
    """The tensor-core path carries activations as fp16 hi/lo pairs: a packed value beyond the fp16 range (|y| > 65504, or NaN)
    cannot be represented. The packing code raises a per-device flag instead of saturating silently; this reads and clears
    it (a blocking 4-byte read on the current stream -- call it where the host waits anyway) and raises."""
    import ctypes
    flag = ctypes.c_int(0)
    check(_lib.lib().sgb_spconv_overflow(ctypes.byref(flag), _stream()), 'sgb_spconv_overflow')
    if flag.value:
        raise _lib.SgbError('sparse convolution: an activation left the fp16 range of the hi/lo split (|y| > 65504 or NaN after '
                            'BatchNorm+ReLU); the tensor-core path cannot represent it -- rescale the checkpoint or run '
                            'SGB_CONV_IMPL=ffma')


class Emit(object):
    """What a producing conv writes besides (or instead of) fp32 rows: the packed rows of ITS CONSUMER's input, i.e.
    relu(y * scale + shift) split into fp16 hi/lo -- the consumer's BatchNorm(eval)+ReLU folded into this epilogue.
    buf/coff: existing packed buffer + channel offset (concat halves) or None for a fresh one (conv_forward stores it
    here); fill: zero the unused half of a last 32-channel chunk. `key` is accepted so that existing callers keep working,
    and is not used."""
    __slots__ = ('scale', 'shift', 'buf', 'coff', 'fill')

    def __init__(self, scale, shift, key=None, buf=None, coff=0, fill=True):
        self.scale, self.shift, self.buf, self.coff, self.fill = scale, shift, buf, coff, fill


def conv_bytes(m_in, Mout, K, Cin, Cout, has_map, has_residual):
    """Algorithmic bytes of one sparse convolution (SURVEY.md 8d): input rows once + weights + map + output rows
    (+ residual rows)."""
    return (4 * m_in * Cin + 4 * K * Cin * Cout + (4 * K * Mout if has_map else 0) + 4 * Mout * Cout +
            (4 * Mout * Cout if has_residual else 0))


def conv_forward(feats, in_stride, in_off, mp, K, Mout, W, Cin, Cout, act=None, residual=None, bias=None, out=None,
                 out_stride=None, out_off=0, packed_in=None, emit=None, want_fp32=True, m_in=None):
    """Thin wrapper over sgb_spconv_forward_tc (wgmma) / sgb_spconv_forward (CUDA cores: SGB_CONV_IMPL=ffma, or shapes
    outside the tensor path). W: WeightPack or [K, Cin, Cout] f32 tensor. act: (scale, shift) or None.
    Tensor path: packed_in = the input already activated + packed (feats may then be None, m_in = its row count);
    emit = Emit(...) makes the epilogue write the consumer's packed input; want_fp32 = False skips the fp32 rows
    (single-consumer intermediates). Returns the fp32 tensor (or None); with emit, (fp32, packed)."""
    if not isinstance(W, WeightPack):
        W = WeightPack(W)
    fused = CONV_IMPL == 'tc' and Cout <= 256 and Cin <= 512
    assert fused or (packed_in is None and emit is None and want_fp32), 'packed I/O needs the tensor-core conv kernel'
    if out is None and want_fp32:
        out = torch.empty((Mout, Cout), dtype=torch.float32, device=(feats if feats is not None else packed_in).device)
        out_stride = Cout
    scale, shift = act if act is not None else (None, None)
    rs, ro = (residual.stride(0), 0) if residual is not None else (0, 0)
    if m_in is None:
        m_in = feats.size(0)
    nbytes = conv_bytes(m_in, Mout, K, Cin, Cout, mp is not None, residual is not None)
    name = ('spconv_tc_kernel' if fused else 'spconv_kernel') + ('' if mp is not None else '(1x1/linear)')
    if fused:
        pk = packed_in if packed_in is not None else act_pack(feats, in_stride, in_off, Cin, act=act, relu=act is not None)
        pk_out, pk_stride, pk_coff, es, eh, fill = None, 0, 0, None, None, 0
        if emit is not None:
            if emit.buf is None:
                emit.buf = torch.empty((Mout, (Cout + 31) // 32 * 32), dtype=torch.float32, device=pk.device)
            pk_out, pk_stride, pk_coff, es, eh, fill = emit.buf, emit.buf.size(1), emit.coff, emit.scale, emit.shift, int(emit.fill)
        with profiler.record(name, nbytes):
            check(
                _lib.lib().sgb_spconv_forward_tc_ex(ptr(pk), pk.size(1), m_in, ptr(mp), K, Mout, ptr(W.tc()), Cin, Cout,
                                                    ptr(residual), rs, ro, ptr(bias), ptr(out), out_stride or 0, out_off,
                                                    ptr(pk_out), pk_stride, pk_coff, ptr(es), ptr(eh), 1, fill, CONV_KERNEL,
                                                    _stream()),
                'sgb_spconv_forward_tc_ex')
        return (out, pk_out) if emit is not None else out
    with profiler.record(name, nbytes):
        check(
            _lib.lib().sgb_spconv_forward(ptr(feats), in_stride, in_off, ptr(mp), K, Mout, ptr(W.kio), Cin, Cout,
                                          ptr(scale), ptr(shift), ptr(residual), rs, ro, ptr(bias), ptr(out),
                                          out_stride, out_off, _stream()), 'sgb_spconv_forward')
    return out


# ---------------------------------------------------------------------------------------------------------
# convolution modules
# ---------------------------------------------------------------------------------------------------------
class _SparseConvBase(SparseModule):

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, bias=True, indice_key=None):
        super().__init__()
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.kernel_size = [kernel_size] * 3 if isinstance(kernel_size, int) else list(kernel_size)
        self.stride = [stride] * 3 if isinstance(stride, int) else list(stride)
        self.padding = [padding] * 3 if isinstance(padding, int) else list(padding)
        self.indice_key = indice_key
        # spconv 2.x layout [out, k0, k1, k2, in] (tools/convert_checkpoint.py:17-19)
        self.weight = nn.Parameter(torch.empty(out_channels, *self.kernel_size, in_channels))
        if bias:
            self.bias = nn.Parameter(torch.zeros(out_channels))
        else:
            self.register_parameter('bias', None)
        self._wt = None
        self.reset_parameters()

    def reset_parameters(self):
        nn.init.kaiming_uniform_(self.weight, a=5**0.5)
        if self.bias is not None:
            fan_in = self.in_channels * self.kernel_size[0] * self.kernel_size[1] * self.kernel_size[2]
            bound = 1 / fan_in**0.5
            nn.init.uniform_(self.bias, -bound, bound)

    def weight_kio(self):
        """[K, Cin, Cout] contiguous copy of the weight, cached until the parameter changes."""
        ver = (self.weight._version, self.weight.data_ptr(), self.weight.device)
        if self._wt is None or self._wt[0] != ver:
            with torch.no_grad():
                w = self.weight.detach().reshape(self.out_channels, -1, self.in_channels).permute(1, 2, 0).contiguous()
            self._wt = (ver, WeightPack(w.float()))
        return self._wt[1]

    def _features(self, x, fuse=None):
        f = x.features
        if f is None:  # a packed-only intermediate (its producer skipped the fp32 rows): the caller hands the packed input
            assert fuse is not None and fuse.get('packed_in') is not None, 'features exist only in packed form'
            return None
        assert f.is_cuda and f.dtype == torch.float32, 'softgroup_b200 sparse convs run on CUDA float32 features'
        if f.stride(-1) != 1:
            f = f.contiguous()
        return f


def _stride0(f):
    return f.stride(0) if f is not None else 0


def _wrap(t, o, fuse):
    """conv_forward result -> SparseConvTensor of the fp32 rows (None when the conv wrote only the packed rows of its
    consumer; those are in fuse['emit'].buf)."""
    t.features = o[0] if fuse.get('emit') is not None else o
    return t


class SubMConv3d(_SparseConvBase):
    """Submanifold 3x3x3 convolution (blocks.py:57-70, softgroup.py:61)."""

    def forward(self, x, act=None, residual=None, out=None, out_stride=None, out_off=0, **fuse):
        assert self.kernel_size == [3, 3, 3], 'only the k=3 submanifold conv of the reference is built'
        f = self._features(x, fuse)
        rb = rulebook(x.indice_dict, self.indice_key, 'subm', x.indices)
        M = x.indices.size(0)
        o = conv_forward(f, _stride0(f), 0, rb['map'], 27, M, self.weight_kio(), self.in_channels, self.out_channels,
                         act=act, residual=residual, bias=self.bias, out=out, out_stride=out_stride, out_off=out_off,
                         m_in=M, **fuse)
        return _wrap(x.replace_feature(None), o, fuse)


class SparseConv3d(_SparseConvBase):
    """k=2 s=2 strided sparse conv (blocks.py:101-107) and, with kernel_size=1, the dense 1x1 (blocks.py:31-41)."""

    def forward(self, x, act=None, residual=None, out=None, out_stride=None, out_off=0, **fuse):
        f = self._features(x, fuse)
        if self.kernel_size == [1, 1, 1]:
            M = x.indices.size(0)
            o = conv_forward(f, _stride0(f), 0, None, 1, M, self.weight_kio(), self.in_channels, self.out_channels,
                             act=act, residual=residual, bias=self.bias, out=out, out_stride=out_stride,
                             out_off=out_off, m_in=M, **fuse)
            return _wrap(x.replace_feature(None), o, fuse)
        assert self.kernel_size == [2, 2, 2] and self.stride == [2, 2, 2] and self.padding == [0, 0, 0], \
            'only the k2 s2 p0 strided conv of the reference is built'
        rb = rulebook(x.indice_dict, self.indice_key, 'down', x.indices, x.spatial_shape)
        Mout = rb['out_indices'].size(0)
        o = conv_forward(f, _stride0(f), 0, rb['map'], 8, Mout, self.weight_kio(), self.in_channels, self.out_channels,
                         act=act, residual=residual, bias=self.bias, out=out, out_stride=out_stride, out_off=out_off,
                         m_in=x.indices.size(0), **fuse)
        t = SparseConvTensor(None, rb['out_indices'], rb['out_shape'], x.batch_size, x.grid, x.indice_dict)
        return _wrap(t, o, fuse)


class SparseInverseConv3d(_SparseConvBase):
    """Inverse of the k2 s2 conv with the same indice_key (blocks.py:114-119): restores its input sites and order."""

    def __init__(self, in_channels, out_channels, kernel_size, indice_key=None, bias=True):
        super().__init__(in_channels, out_channels, kernel_size, bias=bias, indice_key=indice_key)

    def forward(self, x, act=None, residual=None, out=None, out_stride=None, out_off=0, **fuse):
        f = self._features(x, fuse)
        rb = x.find_indice_pair(self.indice_key)
        assert rb is not None and rb['kind'] == 'down', 'SparseInverseConv3d needs the pairs of indice_key %r' % (
            self.indice_key, )
        M = rb['in_indices'].size(0)
        o = conv_forward(f, _stride0(f), 0, rb['inv_map'], 8, M, self.weight_kio(), self.in_channels,
                         self.out_channels, act=act, residual=residual, bias=self.bias, out=out,
                         out_stride=out_stride, out_off=out_off, m_in=x.indices.size(0), **fuse)
        t = SparseConvTensor(None, rb['in_indices'], rb['in_shape'], x.batch_size, x.grid, x.indice_dict)
        return _wrap(t, o, fuse)


# forwards that understand act= / residual= / out= / packed_in= / emit= ...: a subclass that overrides forward with the
# plain spconv signature `forward(self, input)` (the reference's Custom1x1Subm3d, blocks.py:31-41) is an opaque module
for _cls in (SubMConv3d, SparseConv3d, SparseInverseConv3d):
    _cls.forward._sgb_fused = True


def _takes_fusion(m):
    return isinstance(m, _SparseConvBase) and getattr(type(m).forward, '_sgb_fused', False)


# ---------------------------------------------------------------------------------------------------------
# SparseSequential with BN/ReLU -> conv peephole fusion
# ---------------------------------------------------------------------------------------------------------
class SparseSequential(SparseModule):

    def __init__(self, *args, **kwargs):
        super().__init__()
        if len(args) == 1 and isinstance(args[0], OrderedDict):
            for key, module in args[0].items():
                self.add_module(key, module)
        else:
            for idx, module in enumerate(args):
                self.add_module(str(idx), module)
        for name, module in kwargs.items():
            self.add_module(name, module)

    def __getitem__(self, idx):
        if not (-len(self) <= idx < len(self)):
            raise IndexError('index {} is out of range'.format(idx))
        if idx < 0:
            idx += len(self)
        return list(self._modules.values())[idx]

    def __len__(self):
        return len(self._modules)

    def add(self, module, name=None):
        if name is None:
            name = str(len(self._modules))
        self.add_module(name, module)

    @staticmethod
    def _flush(x, pending):
        scale, shift, relu = pending
        if isinstance(x, SparseConvTensor):
            return x.replace_feature(bn_relu_rows(x.features, scale, shift, relu))
        return bn_relu_rows(x, scale, shift, relu)

    def forward(self, input, residual=None, out=None, out_stride=None, out_off=0):
        """residual / out* apply to the LAST sparse conv of the sequence (fused epilogue).

        Tensor-core path: a conv followed inside this sequence by BatchNorm+ReLU+conv writes only the packed rows its
        successor reads (that BatchNorm+ReLU folded into its epilogue, no fp32 rows at all). Fusion across modules is the
        compiled plan's (model/unet_plan.py)."""
        mods = list(self._modules.values())
        conv_idx = [i for i, m in enumerate(mods) if _takes_fusion(m)]
        last_conv = conv_idx[-1] if conv_idx else -1
        fused = CONV_IMPL == 'tc'
        pending = None  # (scale, shift, relu)
        carry = None    # packed input prepared by the previous conv of this sequence for exactly `pending`
        x = input
        for i, m in enumerate(mods):
            is_sparse_in = isinstance(x, SparseConvTensor)
            feats = x.features if is_sparse_in else x
            fusable = feats is None or (feats.is_cuda and feats.dtype == torch.float32)
            if isinstance(m, nn.BatchNorm1d) and fusable and not m.training:
                if pending is not None:
                    x = self._flush(x, pending)
                s, b = fold_bn(m)
                pending = (s, b, False)
                continue
            if isinstance(m, nn.ReLU) and pending is not None and not pending[2]:
                pending = (pending[0], pending[1], True)
                continue
            if _takes_fusion(m):
                act, fuse = None, {}
                if pending is not None:
                    if pending[2]:
                        act = (pending[0], pending[1])
                        if carry is not None:
                            fuse['packed_in'] = carry
                    else:  # BN without ReLU in front of a conv: not fusable into the relu'd input transform
                        x = self._flush(x, pending)
                    pending = None
                carry = None
                nxt = mods[i + 1:i + 4]
                if (fused and is_sparse_in and m.out_channels <= 256 and m.in_channels <= 512 and i != last_conv and
                        len(nxt) == 3 and isinstance(nxt[0], nn.BatchNorm1d) and not nxt[0].training and
                        isinstance(nxt[1], nn.ReLU) and _takes_fusion(nxt[2])):
                    fuse['emit'] = Emit(*fold_bn(nxt[0]))
                    fuse['want_fp32'] = False  # the intermediate never leaves this sequence
                if i == last_conv:
                    x = m(x, act=act, residual=residual, out=out, out_stride=out_stride, out_off=out_off, **fuse)
                else:
                    x = m(x, act=act, **fuse)
                if 'emit' in fuse:
                    carry = fuse['emit'].buf
                continue
            if pending is not None:
                x = self._flush(x, pending)
                pending = None
            if isinstance(m, SparseModule):
                x = m(x)
            elif isinstance(x, SparseConvTensor):
                if isinstance(m, nn.Identity):
                    continue
                if x.indices.shape[0] != 0:
                    x = x.replace_feature(m(x.features))
            else:
                x = m(x)
        if pending is not None:
            x = self._flush(x, pending)
        return x
