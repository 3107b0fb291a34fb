"""Compile the sparse U-Net of the reference-shaped model into a launch plan for the C executor (csrc/unet.cu).

The module path (softgroup_b200/spconv/core.py SparseSequential + model/blocks.py) issues one ctypes call per launch:
~170 per backbone pass at ~40 us of Python each -- more than the GPU needs for most of them. `compile_backbone` walks the
same module tree ONCE (input conv softgroup.py:60-61, UBlock / ResidualBlock blocks.py:44-143, output layer
softgroup.py:65) and emits one `sgb_unet_op` record per launch. It is the one place that fuses ACROSS modules:

  * activations travel packed (fp16 hi/lo) between convolutions; a conv whose output feeds BatchNorm+ReLU+conv writes
    that consumer's packed input from its epilogue (conv1 of a block writes no fp32 rows at all);
  * the residual add of a block is its second conv's epilogue; the last encoder block writes straight into the left half
    of the concat buffer, the inverse conv into the right half (fp32 and packed twins);
  * the 1x1 skip of the first tail block reads the raw concat buffer (one pack pass).

The module path fuses only inside a SparseSequential and packs each block's input with a separate act_pack. That pass
applies the same fmaxf(fmaf(y, scale, shift), 0) to the same fp32 rows as a conv epilogue, so both paths give
bit-identical features (tests/test_gpu_spconv.py::test_plan_equals_module_path).

Per scan `Plan.run` walks the plan in SEGMENTS, one `sgb_unet_run` call each (7 + 1 for the seven-level backbone): a
segment ends where the next launch needs a U-Net level whose rulebook does not exist yet. Opening a level costs one host
wait (the parent count of the strided rulebook); it is taken right after the previous segment's convolutions were enqueued,
so the GPU keeps working through it. One arena per level holds that level's intermediate buffers. `per_launch=True` runs
the same ops one `sgb_unet_run` call each, inside a profiler record named like the module path's launch
(`spconv_tc_kernel`, `act_pack`, `bn_relu`): the per-op timing of exactly the launches the segmented run makes.
"""
import ctypes

import torch
from torch import nn

from .. import profiler
from ..ops import _lib
from ..ops._lib import check
from ..spconv import core
from ..spconv.core import fold_bn

CONV, ACT_PACK, BN_RELU = 1, 2, 4


class UnetOp(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in
                ('kind', 'level_in', 'level_out', 'map_kind', 'K', 'Cin', 'Cout', 'in_buf', 'in_stride', 'in_off', 'pk_in_buf',
                 'pk_in_stride', 'out_buf', 'out_stride', 'out_off', 'pk_out_buf', 'pk_out_stride', 'pk_out_coff', 'pk_fill',
                 'relu', 'res_buf', 'res_stride', 'res_off')] + [(n, ctypes.c_void_p) for n in ('Wp', 'bias', 'scale', 'shift')]


def _r32(c):
    return (c + 31) // 32 * 32


class _F32(object):
    """fp32 rows inside a plan buffer: (buffer id, row stride, column offset, channels)."""
    __slots__ = ('buf', 'stride', 'off', 'C')

    def __init__(self, buf, stride, off, C):
        self.buf, self.stride, self.off, self.C = buf, stride, off, C


class Plan(object):

    def __init__(self):
        self.ops = []        # dicts of UnetOp fields (+ python-side tensors kept alive in self.keep)
        self.bufs = []       # (level, width in floats)
        self.keep = []       # device tensors referenced by raw pointer from the ops
        self.n_levels = 1
        self.key_of_level = {}   # level -> (subm indice_key, down/inverse indice_key of level -> level + 1)
        self.out = None      # _F32 of the result
        self.in_buf = None
        self._c_ops = None

    # ---- building -------------------------------------------------------------------------------------------------
    def new_buf(self, level, width):
        self.bufs.append((level, width))
        self.n_levels = max(self.n_levels, level + 1)
        return len(self.bufs) - 1

    def _dev(self, t):
        if t is None:
            return None
        t = t.detach().contiguous()
        self.keep.append(t)
        return t.data_ptr()

    def op(self, **kw):
        d = dict(kind=0, level_in=0, level_out=0, map_kind=0, K=1, Cin=0, Cout=0, in_buf=-1, in_stride=0, in_off=0, pk_in_buf=-1,
                 pk_in_stride=0, out_buf=-1, out_stride=0, out_off=0, pk_out_buf=-1, pk_out_stride=0, pk_out_coff=0, pk_fill=0,
                 relu=0, res_buf=-1, res_stride=0, res_off=0, Wp=None, bias=None, scale=None, shift=None)
        d.update(kw)
        self.ops.append(d)

    def act_pack(self, level, x, bn=None, into=None, coff=0, relu=None):
        """fp32 rows -> packed buffer under BatchNorm `bn` (+ReLU) or raw. Returns the packed buffer id."""
        scale = shift = None
        if bn is not None:
            scale, shift = fold_bn(bn) if isinstance(bn, nn.Module) else bn
        if relu is None:
            relu = bn is not None
        if into is None:
            into = self.new_buf(level, _r32(x.C))
        fill = core.pack_fill(x.C, self.bufs[into][1], coff)
        self.op(kind=ACT_PACK, level_in=level, level_out=level, Cin=x.C, Cout=fill, in_buf=x.buf, in_stride=x.stride, in_off=x.off,
                pk_out_buf=into, pk_out_stride=self.bufs[into][1], pk_out_coff=coff, relu=int(bool(relu)), scale=self._dev(scale),
                shift=self._dev(shift))
        return into

    def conv(self, m, level_in, level_out, map_kind, pk_in, out=None, emit_bn=None, emit_into=None, emit_coff=0, emit_fill=1,
             emit_slices=None, residual=None):
        """One convolution launch. out: _F32 destination or None; emit_bn: BatchNorm module of the consumer (packed output,
        `emit_slices` = (scale, shift) tensors when only a channel slice of that BatchNorm applies). Returns the packed
        output buffer id (or None)."""
        K = {0: 1, 1: 27, 2: 8, 3: 8}[map_kind]
        w = m.weight_kio()
        pk_out = None
        scale = shift = None
        if emit_bn is not None:
            scale, shift = emit_slices if emit_slices is not None else fold_bn(emit_bn)
            pk_out = emit_into if emit_into is not None else self.new_buf(level_out, _r32(m.out_channels))
        self.op(kind=CONV, level_in=level_in, level_out=level_out, map_kind=map_kind, K=K, Cin=m.in_channels, Cout=m.out_channels,
                pk_in_buf=pk_in, pk_in_stride=self.bufs[pk_in][1],
                out_buf=out.buf if out is not None else -1, out_stride=out.stride if out is not None else 0,
                out_off=out.off if out is not None else 0,
                pk_out_buf=pk_out if pk_out is not None else -1, pk_out_stride=self.bufs[pk_out][1] if pk_out is not None else 0,
                pk_out_coff=emit_coff, pk_fill=int(emit_fill), relu=1,
                res_buf=residual.buf if residual is not None else -1, res_stride=residual.stride if residual is not None else 0,
                res_off=residual.off if residual is not None else 0,
                Wp=self._dev(w.tc()), bias=self._dev(m.bias), scale=self._dev(scale), shift=self._dev(shift))
        return pk_out

    # ---- per scan ---------------------------------------------------------------------------------------------------
    def finalize(self):
        arr = (UnetOp * len(self.ops))()
        for i, d in enumerate(self.ops):
            for k, v in d.items():
                setattr(arr[i], k, v)
        self._c_ops = arr
        # segments of consecutive ops that need no level beyond the ones already opened: (first op, last op + 1, levels that
        # must be open before it runs). Opening level k = strided rulebook of level k-1 (a host wait for the parent count)
        # + submanifold rulebook of level k. The wait happens while the previous segment's convolutions are still running.
        self.segments = []
        opened, start = 0, 0
        for i, d in enumerate(self.ops):
            need = max(d['level_in'], d['level_out'])
            if need > opened:
                if i > start:
                    self.segments.append((start, i, opened))
                start, opened = i, need
        self.segments.append((start, len(self.ops), opened))

    @staticmethod
    def _record_of(d, M):
        """(profiler name, algorithmic bytes) of op `d` at the row counts M[level]."""
        Min, Mout = M[d['level_in']], M[d['level_out']]
        if d['kind'] == CONV:
            name = 'spconv_tc_kernel' if d['map_kind'] else 'spconv_tc_kernel(1x1/linear)'
            return name, core.conv_bytes(Min, Mout, d['K'], d['Cin'], d['Cout'], d['map_kind'] != 0, d['res_buf'] >= 0)
        return ('act_pack' if d['kind'] == ACT_PACK else 'bn_relu'), 8 * Min * d['Cin']

    def run(self, x, per_launch=False):
        """x: SparseConvTensor (fp32 features [M0, Cin]) -> fp32 features [M0, Cout] of the compiled stack.
        per_launch: one sgb_unet_run call and one profiler record per op instead of one call per segment."""
        assert self._c_ops is not None
        feats = x.features.contiguous()
        dev = feats.device
        L = self.n_levels
        M = [0] * L
        subm, down, inv = [None] * L, [None] * L, [None] * L
        level_idx = [None] * L   # (indices, spatial shape) per level
        arenas = []
        ptrs = [0] * len(self.bufs)
        bufs_of_level = [[] for _ in range(L)]
        for b, (level, width) in enumerate(self.bufs):
            bufs_of_level[level].append((b, width))

        def open_level(k):
            if k == 0:
                indices, shape = x.indices, x.spatial_shape
            else:
                rd = core.rulebook(x.indice_dict, self.key_of_level.get(k - 1, (None, None))[1], 'down', *level_idx[k - 1])
                down[k - 1], inv[k - 1] = rd['map'], rd['inv_map']
                indices, shape = rd['out_indices'], rd['out_shape']
            level_idx[k] = (indices, shape)
            M[k] = indices.size(0)
            subm[k] = core.rulebook(x.indice_dict, self.key_of_level.get(k, (None, None))[0], 'subm', indices)['map']
            total, offs = 0, []
            for b, width in bufs_of_level[k]:
                offs.append(total)
                total += (M[k] * width + 63) // 64 * 64
            arena = torch.empty(max(total, 1), dtype=torch.float32, device=dev)  # one arena per level
            arenas.append(arena)
            for (b, width), o in zip(bufs_of_level[k], offs):
                ptrs[b] = arena.data_ptr() + 4 * o

        opened = -1
        lib = _lib.lib()
        ptrs[self.in_buf] = feats.data_ptr()
        # the argument arrays live for the whole run and are updated in place when a level opens (they were rebuilt from
        # Python lists for every segment: ~0.3 ms of host time per scan)
        c_bufs = (ctypes.c_void_p * len(ptrs))()
        c_subm, c_down, c_inv = (ctypes.c_void_p * L)(), (ctypes.c_void_p * L)(), (ctypes.c_void_p * L)()
        c_M = (ctypes.c_int * L)()
        c_bufs[self.in_buf] = ptrs[self.in_buf]
        stream = _lib.stream()
        op_size = ctypes.sizeof(UnetOp)
        for (i0, i1, need) in self.segments:
            while opened < need:
                opened += 1
                open_level(opened)
                k = opened
                for b, _w in bufs_of_level[k]:
                    c_bufs[b] = ptrs[b] or None
                ptrs[self.in_buf] = feats.data_ptr()  # (open_level(0) gave the input buffer an arena slot: the caller's rows win)
                c_bufs[self.in_buf] = ptrs[self.in_buf]
                c_M[k] = M[k]
                c_subm[k] = subm[k].data_ptr() if subm[k] is not None else None
                if k > 0:
                    c_down[k - 1] = down[k - 1].data_ptr() if down[k - 1] is not None else None
                    c_inv[k - 1] = inv[k - 1].data_ptr() if inv[k - 1] is not None else None
            for j0, j1 in ([(i, i + 1) for i in range(i0, i1)] if per_launch else [(i0, i1)]):
                name, nbytes = self._record_of(self.ops[j0], M) if per_launch else ('unet_run', 0)
                seg = ctypes.cast(ctypes.byref(self._c_ops, j0 * op_size), ctypes.c_void_p)
                with profiler.record(name, nbytes):
                    check(lib.sgb_unet_run(seg, j1 - j0, c_bufs, c_subm, c_down, c_inv, c_M, L, stream), 'sgb_unet_run')
        o = self.out
        level, width = self.bufs[o.buf]
        base = ptrs[o.buf]
        arena = arenas[level]
        off = (base - arena.data_ptr()) // 4
        res = arena[off:off + M[level] * width].view(M[level], width)[:, o.off:o.off + o.C]
        res._sgb_arenas = arenas  # the views keep their arena alive; keep the others until the result dies as well
        return res


# ---------------------------------------------------------------------------------------------------------------------
# tree walk
# ---------------------------------------------------------------------------------------------------------------------
def _block(plan, blk, level, x, x_packed, next_bn, out=None):
    """ResidualBlock (blocks.py:44-79). x: _F32 input, x_packed: {bn module: packed buf}. Returns (_F32 y, {bn: packed})."""
    bn1, conv1, bn2, conv2 = blk.conv_branch[0], blk.conv_branch[2], blk.conv_branch[3], blk.conv_branch[5]
    C = conv2.out_channels
    first = blk.i_branch[0]
    if isinstance(first, nn.Identity):
        skip = x
    else:  # Custom1x1Subm3d on the raw input (blocks.py:31-41)
        pk_raw = plan.act_pack(level, x)
        sb = plan.new_buf(level, C)
        skip = _F32(sb, C, 0, C)
        plan.conv(first, level, level, 0, pk_raw, out=skip)
    pk1 = x_packed.get(bn1)
    if pk1 is None:
        pk1 = plan.act_pack(level, x, bn=bn1)
    pk2 = plan.conv(conv1, level, level, 1, pk1, out=None, emit_bn=bn2)
    if out is None:
        ob = plan.new_buf(level, C)
        out = _F32(ob, C, 0, C)
    pk_y = plan.conv(conv2, level, level, 1, pk2, out=out, emit_bn=next_bn, residual=skip)
    return out, ({next_bn: pk_y} if next_bn is not None else {})


def _ublock(plan, ub, level, x, x_packed, next_bn):
    """UBlock (blocks.py:82-143). Returns (_F32 output, {bn: packed})."""
    deeper = len(ub.nPlanes) > 1
    C = ub.nPlanes[0]
    blocks = list(ub.blocks._modules.values())
    plan.key_of_level[level] = (blocks[0].conv_branch[2].indice_key, ub.conv[2].indice_key if deeper else None)
    cat = None
    if deeper:
        cb = plan.new_buf(level, 2 * C)
        cat = _F32(cb, 2 * C, 0, 2 * C)
    y, yp = x, x_packed
    for i, blk in enumerate(blocks):
        last = i == len(blocks) - 1
        nb = blocks[i + 1].conv_branch[0] if not last else (ub.conv[0] if deeper else next_bn)
        # the last encoder block writes its fp32 rows straight into the left half of the concat buffer
        y, yp = _block(plan, blk, level, y, yp, nb, out=_F32(cat.buf, 2 * C, 0, C) if (last and deeper) else None)
    if not deeper:
        return y, yp
    tail = list(ub.blocks_tail._modules.values())
    tail_bn = tail[0].conv_branch[0]
    ts, tb = fold_bn(tail_bn)
    pk_cat = plan.new_buf(level, _r32(2 * C))
    plan.act_pack(level, y, bn=(ts[:C], tb[:C]), into=pk_cat, coff=0, relu=True)
    # strided conv (blocks.py:101-107): consumer = first BatchNorm of the next level
    C2 = ub.nPlanes[1]
    db = plan.new_buf(level + 1, C2)
    d = _F32(db, C2, 0, C2)
    inner_first = list(ub.u.blocks._modules.values())[0].conv_branch[0]
    pk_d = plan.conv(ub.conv[2], level, level + 1, 2, yp[ub.conv[0]], out=d, emit_bn=inner_first)
    u_out, u_pk = _ublock(plan, ub.u, level + 1, d, {inner_first: pk_d}, ub.deconv[0])
    # inverse conv (blocks.py:114-119) into the right half of the concat buffer, fp32 and packed
    plan.conv(ub.deconv[2], level + 1, level, 3, u_pk[ub.deconv[0]], out=_F32(cat.buf, 2 * C, C, C), emit_bn=tail_bn,
              emit_into=pk_cat, emit_coff=C, emit_fill=0, emit_slices=(ts[C:], tb[C:]))
    y, yp = cat, {tail_bn: pk_cat}
    for i, blk in enumerate(tail):
        nb = tail[i + 1].conv_branch[0] if i + 1 < len(tail) else next_bn
        y, yp = _block(plan, blk, level, y, yp, nb)
    return y, yp


def compile_backbone(input_conv, unet, output_layer):
    """input_conv: SparseSequential(SubMConv3d) (softgroup.py:60-61) or None; unet: UBlock; output_layer:
    SparseSequential(BatchNorm1d, ReLU) (softgroup.py:65) or None. Returns a finalized Plan."""
    plan = Plan()
    first_bn = list(unet.blocks._modules.values())[0].conv_branch[0]
    if input_conv is not None:
        conv0 = input_conv[0]
        plan.in_buf = plan.new_buf(0, conv0.in_channels)
        x = _F32(plan.in_buf, conv0.in_channels, 0, conv0.in_channels)
        pk_in = plan.act_pack(0, x)
        C0 = conv0.out_channels
        ob = plan.new_buf(0, C0)
        y = _F32(ob, C0, 0, C0)
        pk_y = plan.conv(conv0, 0, 0, 1, pk_in, out=y, emit_bn=first_bn)
        yp = {first_bn: pk_y}
    else:
        C0 = unet.nPlanes[0]
        plan.in_buf = plan.new_buf(0, C0)
        y, yp = _F32(plan.in_buf, C0, 0, C0), {}
    y, yp = _ublock(plan, unet, 0, y, yp, None)
    if output_layer is not None:
        bn = output_layer[0]
        s, b = fold_bn(bn)
        ob = plan.new_buf(0, y.C)
        plan.op(kind=BN_RELU, level_in=0, level_out=0, Cin=y.C, in_buf=y.buf, in_stride=y.stride, in_off=y.off, out_buf=ob, out_stride=y.C,
                out_off=0, relu=1, scale=plan._dev(s), shift=plan._dev(b))
        y = _F32(ob, y.C, 0, y.C)
    plan.out = y
    plan.finalize()
    return plan
