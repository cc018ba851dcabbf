"""LSTM2's input projection (proj_tc.cu) splits its work statically: 5 weight slabs of 256 columns times contiguous ranges of
128-row h1 tiles, one CTA per (slab, range), ranges = min(SMs // 5, tiles).  A batch of n sites has bp = n rounded up to 128
rows per time step and 33 * bp / 128 tiles.

On H100 (132 SMs) that is 26 ranges:
  * 600 sites: bp = 640 -> 165 tiles = 26 * 6 + 9 -> 9 ranges of 7 tiles and 17 of 6;
  * its pieces 256 sites (bp = 256 -> 66 tiles = 26 * 2 + 14) and 344 sites (bp = 384 -> 99 tiles = 26 * 3 + 21) split unevenly
    too, each in its own way.
Every site's output must not depend on how the batch was cut.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_uneven_tile_ranges_match_batch_pieces():
    from clair3_b200 import synth
    from clair3_b200.model import Clair3_P
    from oracle import clair3_oracle as orc

    sd = synth.pileup_state_dict(False, seed=11)
    x = synth.pileup_inputs(600, seed=11)
    m = Clair3_P(add_indel_length=False, predict=True, input_channels=18)
    m.to(torch.device("cuda"))
    m.eval()
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    whole = m(torch.from_numpy(x).cuda()).cpu().numpy()
    pieces = np.concatenate([m(torch.from_numpy(x[a:b]).cuda()).cpu().numpy() for a, b in ((0, 256), (256, 600))])
    assert np.isfinite(whole).all()
    assert np.abs(whole - pieces).max() <= 1e-5
    ref = orc.pileup_forward(sd, x, False)
    assert np.abs(whole - ref).max() < 2e-2
