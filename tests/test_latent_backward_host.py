"""The host's choice of a one-pass backward for a latent site (b2_latent_normal_backward): loc's and scale's
gradients are reduced in one pass exactly when they are summed over the same groups of elements.  Checked on
the CPU against the groups that the per-element index math (unravel: flat index -> operand offsets) forms."""
import ctypes
import itertools

import numpy as np
import pytest

import hostcheck
from pyro_b200 import _native as N


def _job(shape, st_loc, st_scale):
    j = N.b2_latent_job()
    j.dtype, j.ndim = N.B2_F32, len(shape)
    for d, (n, a, b) in enumerate(zip(shape, st_loc, st_scale)):
        j.shape[d], j.loc_stride[d], j.scale_stride[d] = n, a, b
    return j


def _groups(shape, st):
    """Partition of the flat element indices by the operand offset each one reads (unravel, row-major)."""
    g = {}
    for i, idx in enumerate(itertools.product(*[range(n) for n in shape])):
        g.setdefault(int(np.dot(idx, st)), []).append(i)
    return sorted(g.values())


def _stored_strides(shape, bcast):
    """Contiguous strides of the operand's stored shape, 0 on its broadcast dims (as torch's expand gives)."""
    st, c = [0] * len(shape), 1
    for d in reversed(range(len(shape))):
        if not bcast[d]:
            st[d] = c
            c *= shape[d]
    return st


SHAPES = [(64, 1, 32), (64, 1), (4, 3, 5), (2, 1, 3, 1), (7,), (1, 1)]


@pytest.mark.parametrize("shape", SHAPES)
def test_same_reduction_matches_unravel_groups(shape):
    L = hostcheck.lib()
    L.b2h_latent_same_reduction.argtypes = [ctypes.POINTER(N.b2_latent_job)]
    nd = len(shape)
    for bl in itertools.product([False, True], repeat=nd):
        for bs in itertools.product([False, True], repeat=nd):
            st_l, st_s = _stored_strides(shape, bl), _stored_strides(shape, bs)
            # a size-1 dim may carry any stride: it never moves the offset
            st_s = [7 if (n == 1 and b) else s for n, b, s in zip(shape, bs, st_s)]
            got = L.b2h_latent_same_reduction(ctypes.byref(_job(shape, st_l, st_s)))
            want = _groups(shape, st_l) == _groups(shape, st_s)
            assert got == int(want), (shape, st_l, st_s, got)


def test_same_reduction_rejects_what_the_backward_rejects():
    L = hostcheck.lib()
    L.b2h_latent_same_reduction.argtypes = [ctypes.POINTER(N.b2_latent_job)]
    assert L.b2h_latent_same_reduction(ctypes.byref(_job((0, 3), (0, 1), (0, 1)))) < 0
    assert L.b2h_latent_same_reduction(ctypes.byref(_job((300, 300), (0, 1), (0, 1)))) < 0
