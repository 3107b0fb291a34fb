"""Thin helpers the forward touches (reference: softgroup/util/utils.py:157-173 cuda_cast,
softgroup/util/fp16.py:27-66 force_fp32)."""
import functools

import torch


def cuda_cast(func):
    """Move every tensor argument to the current CUDA device (non_blocking: collated batches are pinned)."""

    @functools.wraps(func)
    def wrapper(*args, **kwargs):
        new_args = [x.cuda(non_blocking=True) if isinstance(x, torch.Tensor) else x for x in args]
        new_kwargs = {k: (v.cuda(non_blocking=True) if isinstance(v, torch.Tensor) else v) for k, v in kwargs.items()}
        return func(*new_args, **new_kwargs)

    return wrapper


def force_fp32(apply_to=None, out_fp16=False):
    """The GPU path computes in fp32 throughout; kept so decorated methods read like the reference's.
    Half inputs (from a caller using autocast) are widened."""

    def deco(old_func):

        @functools.wraps(old_func)
        def new_func(*args, **kwargs):
            cast = lambda v: v.float() if isinstance(v, torch.Tensor) and v.dtype == torch.half else v  # noqa: E731
            return old_func(*[cast(a) for a in args], **{k: cast(v) for k, v in kwargs.items()})

        return new_func

    return deco
