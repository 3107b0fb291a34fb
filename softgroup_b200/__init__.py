"""softgroup_b200 -- H100 (sm_90a) implementation of SoftGroup's per-scan inference hot path.

Layout: csrc/ (CUDA kernels + C ABI, built into libsgb200.so), ops/ (the reference's softgroup.ops binding
surface), spconv/ (the spconv-shaped surface the reference model touches), model/ (SoftGroup nn.Module mirror),
synth.py (synthetic scans), util/.
"""
import sys

__version__ = '0.1.0'


def install_as_reference_backends(torch2_compat=False):
    """Register this package's modules under the names the UNMODIFIED reference imports, so that
    `softgroup/model/*.py` and `tools/test.py` of thangvubk/SoftGroup run on these kernels:
        import spconv.pytorch as spconv          -> softgroup_b200.spconv.pytorch
        from spconv.pytorch.modules import ...   -> softgroup_b200.spconv.pytorch.modules
        from . import ops  (softgroup/ops/functions.py:4, the compiled extension) is bypassed by providing
        `softgroup.ops` = softgroup_b200.ops
    Call before importing `softgroup`. See INTEGRATION.md.
    torch2_compat: the reference indexes the CPU cluster tensor with a CUDA mask (softgroup.py:570), which PyTorch >= 2
    rejects; with this switch `bfs_cluster` returns its CPU result as a tensor subclass that copies CUDA indices to the host
    first (ops/functions.py:HostIndexTensor), so the unmodified reference model runs on a current PyTorch."""
    from . import ops
    from .ops import functions as _f
    _f.TORCH2_COMPAT = bool(torch2_compat)
    from . import spconv as sp
    from .spconv import pytorch as sp_pt
    sys.modules.setdefault('spconv', sp)
    sys.modules.setdefault('spconv.pytorch', sp_pt)
    sys.modules.setdefault('spconv.pytorch.modules', sp_pt.modules)
    sys.modules.setdefault('softgroup.ops', ops)
    return ops, sp
