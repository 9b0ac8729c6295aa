"""The epilogue warpgroup of the wgmma GEMM (csrc/conv_gemm.cuh) drains one tile while the consumers compute the
next.  These cases run many tiles per CTA, where the consumers can get a whole main loop ahead of the epilogue, and
check them the way tests/test_gpu_gemm_cluster.py does: against fp64, and bitwise against the same rows computed at
another position (the input shifted by 128 rows, or by whole images).
"""
import pytest

import test_gpu_gemm_cluster as cluster
from test_gpu_gemm import ACT_GELU

pytestmark = pytest.mark.gpu


def test_one_kstep_linear_many_tiles(engine):
    """K = 64 (one k-step per tile, split weights, GELU), 1407 -> 1408 M tiles: ~10 tiles per CTA, each main loop far
    shorter than its epilogue, so the consumers wait on the epilogue at every tile."""
    cluster.test_linear_rows_same_on_either_rank(engine, 180001, 64, 128, ACT_GELU, 1)


def test_fused_residual_many_tiles(engine):
    """The fused residual update over 2344 -> 2345 M tiles x 3 N tiles."""
    cluster.test_fused_residual_same_on_either_rank(engine, 300001)


def test_conv2_shape_many_images(engine):
    """conv2 of VGGish (48 x 32, 64 -> 128 channels, 9 k-steps, 2x2 max-pool) over 256 images: 3072 tiles.  An image
    is 12 tiles, so the one-image shift keeps each tile on its rank but moves it to another work unit."""
    cluster.test_conv_rows_same_on_either_rank(engine, 256, 48, 32, 64, 128, True, 1, 1)
