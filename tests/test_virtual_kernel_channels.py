"""Real<->virtual kernel, one instantiation per channel count: distegnn_virtual_layer_fwd and its deterministic twin are
compiled for every C in 1..DISTEGNN_MAX_CHANNELS, each with its own index arithmetic, pool and sum loops and per-node
geometry.  Every C runs, in both modes and with and without FLAG_LAST, on

  * a layout of small and large graphs with N a multiple of no tile's node count (64 // C for every C), so that tiles
    straddle graphs (one or many boundaries, empty graph ids), the G cache is reloaded between a warpgroup's tiles, and
    the last tile is ragged;
  * a single node.

The checks are test_virtual_kernel_tiling.check: against the fp32-FMA twin over the tensor and against float64 row by
row and graph by graph; the deterministic mode also at grid caps 1 and 7, bit for bit (test_forward_det_tiling)."""
import pytest
import torch

from tests import test_virtual_kernel_tiling as vk
from tests.test_forward_det_tiling import det_virtual

pytestmark = pytest.mark.gpu

CHANNELS = list(range(1, 17))
KERNELS = {"default": vk.production, "deterministic": det_virtual}


def straddling_sizes():
    """Graph sizes: tiny graphs and empty ids around a few graphs of hundreds of nodes; N is a multiple of no 64 // C."""
    g = torch.Generator().manual_seed(7)
    sizes = [1, 0, 2, 3, 1, 5, 0, 0, 7, 9, 1, 13, 700, 1, 2, 0, 31, 33, 17, 4, 900, 3, 1, 65, 63, 2, 0, 1]
    sizes += torch.randint(0, 12, (40,), generator=g).tolist() + [1_000]
    n = sum(sizes)
    tns = {64 // c for c in CHANNELS}
    while any(n % tn == 0 for tn in tns):
        sizes[-1] += 1
        n += 1
    return sizes


@pytest.mark.parametrize("C", CHANNELS)
@pytest.mark.parametrize("flags", vk.FLAGS)
@pytest.mark.parametrize("mode", list(KERNELS))
def test_tiles_straddle_graphs_and_the_last_tile_is_ragged(C, flags, mode):
    sizes = straddling_sizes()
    batch = vk.batch_of_sizes(sizes)
    assert batch.numel() % (64 // C) != 0
    vk.check(batch, len(sizes), C, flags, seed=100 + C, kernel=KERNELS[mode])


@pytest.mark.parametrize("C", CHANNELS)
@pytest.mark.parametrize("flags", vk.FLAGS)
@pytest.mark.parametrize("mode", list(KERNELS))
def test_a_single_node(C, flags, mode):
    vk.check(torch.zeros(1, dtype=torch.int64), 1, C, flags, seed=200 + C, kernel=KERNELS[mode])
