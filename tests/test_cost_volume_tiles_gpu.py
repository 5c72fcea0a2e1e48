"""Tile-edge parity of the fused cost-volume kernel: the shortest march, a last 16-row tile with a single valid row.  Needs an
H100."""
import pytest

from tests.helpers import compare_volumes
from tests.test_cost_volume_gpu import _run

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("cfg", [(1, 4, 64, 67, 180, 43), (2, 3, 16, 51, 123, 44)])
def test_single_valid_row_in_last_tile_against_oracle(cfg):
    """H = 16 k + 3: the last tile holds rows H-3 .. H-1, of which only H-3 is valid (pixels with v >= H - 2 are invalid), so
    every frame's march over that tile is the minimal 5 steps.  W % 4 == 0 takes the TMA windows, the odd W the global
    gather with scalar stores."""
    from oracle import cost_volume_oracle as O
    from monorec_b200.synthetic import make_inputs
    B, F, D, H, W, seed = cfg
    data = make_inputs(B, F, H, W, seed=seed)
    ref_cv, ref_sf = O.cost_volume_torch(data, steps=D)
    cv, sf = _run(data, steps=D)
    print(cfg, compare_volumes(cv, sf, ref_cv, ref_sf))
