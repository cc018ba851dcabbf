"""Each packed weight image holds exactly what its forward path reads (``pytest -m gpu`` on an H100).

``weight_blob(0)`` is everything the default fp16 tensor-core forward reads and ``weight_blob(1)`` what only the fp32 path
(precision=1) reads; the fp32 path reads both.  A rank that receives the images by broadcast relies on this: with image 0
alone it must compute the default-precision outputs bit for bit.  Model B is loaded with zeros of the same shapes and
receives model A's images by a device-to-device copy, the way a broadcast writes them.
"""
import numpy as np
import pytest
import torch

from clair3_b200 import synth
from clair3_b200.model import Clair3_F, Clair3_P
from clair3_b200.sharding import _DevBlob, zeros_like_state_dict

pytestmark = pytest.mark.gpu


def _load(cls, sd, add_indel, channels):
    m = cls(add_indel_length=add_indel, predict=True, input_channels=channels)
    m.to(torch.device("cuda"))
    m.load_state_dict({k: torch.as_tensor(np.asarray(v)) for k, v in sd.items()})
    return m


def _copy_image(src, dst, which):
    """Copies image `which` of model src over dst's, device to device, through tensors aliasing the library's images."""
    (ps, ns), (pd, nd) = src.weight_blob(which), dst.weight_blob(which)
    assert ns == nd
    torch.as_tensor(_DevBlob(pd, nd), device=dst._device).copy_(torch.as_tensor(_DevBlob(ps, ns), device=src._device))
    torch.cuda.synchronize()


@pytest.mark.parametrize("add_indel", [False, True])
@pytest.mark.parametrize("kind", ["pileup", "fa"])
def test_image0_carries_the_tensor_core_forward(kind, add_indel):
    if kind == "pileup":
        cls, channels = Clair3_P, synth.P_CHANNELS
        sd = synth.pileup_state_dict(add_indel, seed=21)
        x = torch.from_numpy(synth.pileup_inputs(300, seed=21)).cuda()
    else:
        cls, channels = Clair3_F, 8
        sd = synth.fa_state_dict(add_indel, channels=channels, seed=22)
        x = torch.from_numpy(synth.fa_inputs(40, depth=89, channels=channels, seed=22)).cuda()
    a = _load(cls, sd, add_indel, channels)
    b = _load(cls, zeros_like_state_dict({k: np.shape(v) for k, v in sd.items()}), add_indel, channels)
    for which in (0, 1):
        assert b.weight_blob(which)[1] == a.weight_blob(which)[1]

    _copy_image(a, b, 0)
    assert torch.equal(b(x), a(x))

    a.set_option("precision", 1)
    b.set_option("precision", 1)
    ya = a(x)
    assert not torch.equal(b(x), ya)
    _copy_image(a, b, 1)
    assert torch.equal(b(x), ya)
