"""Module tree of the reference's softgroup/model/blocks.py (MLP :9-27, Custom1x1Subm3d :31-41, ResidualBlock
:44-79, UBlock :82-143) with IDENTICAL parameter names and shapes, running on libsgb200 kernels.

What changes underneath (results equal within fp32 rounding):
  * BatchNorm1d(eval)+ReLU in front of a sparse conv is folded into that conv's input transform;
  * the residual add of ResidualBlock is the second conv's epilogue;
  * the decoder's SparseInverseConv3d writes straight into the right half of the [M, 2C] concat buffer;
  * MLP heads run through the same kernel (K=1 identity map) with bias / BN / ReLU fused.

Each block packs its own input here. On the tensor-core path SoftGroup runs the U-Net as a compiled plan instead
(model/unet_plan.py), which fuses across blocks too; both give bit-identical features.
"""
from collections import OrderedDict

import torch
from torch import nn

from .. import spconv
from ..spconv import SparseModule, conv_forward, fold_bn
from ..spconv.core import WeightPack


class MLP(nn.Sequential):

    def __init__(self, in_channels, out_channels, norm_fn=None, num_layers=2):
        modules = []
        for _ in range(num_layers - 1):
            modules.append(nn.Linear(in_channels, in_channels))
            if norm_fn:
                modules.append(norm_fn(in_channels))
            modules.append(nn.ReLU())
        modules.append(nn.Linear(in_channels, out_channels))
        super().__init__(*modules)
        self._cache = {}

    def init_weights(self):
        for m in self.modules():
            if isinstance(m, nn.Linear):
                nn.init.xavier_uniform_(m.weight)
                nn.init.constant_(m.bias, 0)
        nn.init.normal_(self[-1].weight, 0, 0.01)
        nn.init.constant_(self[-1].bias, 0)

    def _wt(self, lin):
        ver = (lin.weight._version, lin.weight.data_ptr())
        hit = self._cache.get(id(lin))
        if hit is None or hit[0] != ver:
            hit = (ver, WeightPack(lin.weight.detach().t().contiguous().unsqueeze(0).float()))  # [1, Cin, Cout]
            self._cache[id(lin)] = hit
        return hit[1]

    def _unit(self, C, device):
        key = ('unit', C, str(device))
        if key not in self._cache:
            self._cache[key] = (torch.ones(C, device=device), torch.zeros(C, device=device))
        return self._cache[key]

    def forward(self, x):
        if not (x.is_cuda and x.dtype == torch.float32) or self.training or torch.is_grad_enabled():
            return super().forward(x)  # training / autograd path stays plain PyTorch (out of scope here)
        x = x.contiguous()
        act = None
        mods = list(self)
        i = 0
        while i < len(mods):
            m = mods[i]
            if isinstance(m, nn.Linear):
                x = conv_forward(x, x.stride(0), 0, None, 1, x.size(0), self._wt(m), m.in_features, m.out_features,
                                 act=act, bias=m.bias)
                act = None
            elif isinstance(m, nn.BatchNorm1d):
                act = fold_bn(m)
                assert isinstance(mods[i + 1], nn.ReLU)
                i += 1
            elif isinstance(m, nn.ReLU):
                act = self._unit(x.size(1), x.device)
            else:
                raise RuntimeError('unexpected module in MLP: %r' % (m, ))
            i += 1
        assert act is None
        return x


class Custom1x1Subm3d(spconv.SparseConv3d):
    """1x1 conv as a dense per-row contraction (blocks.py:31-41 uses torch.mm for the same thing)."""

    def forward(self, input, **kw):
        out_tensor = super().forward(input, **kw)
        out_tensor.indice_dict = input.indice_dict
        out_tensor.grid = input.grid
        return out_tensor

    forward._sgb_fused = True


class ResidualBlock(SparseModule):

    def __init__(self, in_channels, out_channels, norm_fn, indice_key=None):
        super().__init__()
        if in_channels == out_channels:
            self.i_branch = spconv.SparseSequential(nn.Identity())
        else:
            self.i_branch = spconv.SparseSequential(
                Custom1x1Subm3d(in_channels, out_channels, kernel_size=1, bias=False))
        self.conv_branch = spconv.SparseSequential(
            norm_fn(in_channels), nn.ReLU(),
            spconv.SubMConv3d(in_channels, out_channels, kernel_size=3, padding=1, bias=False, indice_key=indice_key),
            norm_fn(out_channels), nn.ReLU(),
            spconv.SubMConv3d(out_channels, out_channels, kernel_size=3, padding=1, bias=False,
                              indice_key=indice_key))

    def forward(self, input):
        skip = self.i_branch(input).features
        # output.features + i_branch(identity).features (blocks.py:75-76), as the second conv's epilogue
        return self.conv_branch(input, residual=skip)


class UBlock(nn.Module):

    def __init__(self, nPlanes, norm_fn, block_reps, block, indice_key_id=1):
        super().__init__()
        self.nPlanes = nPlanes
        blocks = {
            'block{}'.format(i): block(nPlanes[0], nPlanes[0], norm_fn, indice_key='subm{}'.format(indice_key_id))
            for i in range(block_reps)
        }
        self.blocks = spconv.SparseSequential(OrderedDict(blocks))
        if len(nPlanes) > 1:
            self.conv = spconv.SparseSequential(
                norm_fn(nPlanes[0]), nn.ReLU(),
                spconv.SparseConv3d(nPlanes[0], nPlanes[1], kernel_size=2, stride=2, bias=False,
                                    indice_key='spconv{}'.format(indice_key_id)))
            self.u = UBlock(nPlanes[1:], norm_fn, block_reps, block, indice_key_id=indice_key_id + 1)
            self.deconv = spconv.SparseSequential(
                norm_fn(nPlanes[1]), nn.ReLU(),
                spconv.SparseInverseConv3d(nPlanes[1], nPlanes[0], kernel_size=2, bias=False,
                                           indice_key='spconv{}'.format(indice_key_id)))
            blocks_tail = {}
            for i in range(block_reps):
                blocks_tail['block{}'.format(i)] = block(nPlanes[0] * (2 - i), nPlanes[0], norm_fn,
                                                         indice_key='subm{}'.format(indice_key_id))
            self.blocks_tail = spconv.SparseSequential(OrderedDict(blocks_tail))

    def forward(self, input):
        output = self.blocks(input)
        if len(self.nPlanes) > 1:
            C = self.nPlanes[0]
            M = output.features.size(0)
            # torch.cat((identity.features, output_decoder.features), dim=1) (blocks.py:140) without the cat:
            cat = torch.empty((M, 2 * C), dtype=output.features.dtype, device=output.features.device)
            cat[:, :C] = output.features
            output_decoder = self.u(self.conv(output))
            self.deconv(output_decoder, out=cat, out_stride=2 * C, out_off=C)
            output = self.blocks_tail(output.replace_feature(cat))
        return output
