"""The TF32 emulation of the reference on a GPU (tests/tf32_reference.py), on the CPU: the rounding itself, and that it
reaches every convolution of the oracle inside the block and none outside it."""
import torch

from oracle import dvc_oracle as O
from tf32_reference import round_tf32, tf32_conv_operands


def test_round_tf32_values():
    u = 2.0 ** -11
    t = torch.tensor([1.0, 1 + u, 1 + 3 * u, 1 + 2 * u + 2 ** -20, -(1 + 3 * u), 3.0, 0.0], dtype=torch.float64)
    # ties (1 + u, 1 + 3u) go to the even 11-bit neighbour; above a tie rounds up
    want = [1.0, 1.0, 1 + 4 * u, 1 + 2 * u, -(1 + 4 * u), 3.0, 0.0]
    assert round_tf32(t).tolist() == want
    x = torch.randn(1000, dtype=torch.float64, generator=torch.Generator().manual_seed(0)) * 1e3
    r = round_tf32(x)
    assert ((r - x).abs() <= x.abs() * 2.0 ** -11).all()
    assert torch.equal(round_tf32(r), r)


def test_emulation_is_scoped_to_the_block():
    from oracle.weights import make_state_dict

    sd = O._cast(make_state_dict("vgg", seed=0), torch.float64)
    x = torch.rand(1, 3, 32, 32, dtype=torch.float64, generator=torch.Generator().manual_seed(1))
    exact = O.vgg19_forward(sd, x, ("r12",))[0]
    with tf32_conv_operands():
        emulated = O.vgg19_forward(sd, x, ("r12",))[0]
    again = O.vgg19_forward(sd, x, ("r12",))[0]
    assert torch.equal(exact, again)
    d = (emulated - exact).abs().max().item() / exact.abs().max().item()
    assert 0 < d < 1e-2, d
