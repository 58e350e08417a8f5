"""CUDA HiFiGAN generator vs golden fixtures (reference outputs) and vs the oracle at full width.
north_star tolerance: waveform within 1e-4 RMS.  The decoder convs run on the wgmma 3xTF32 kernel (fp32
accumulate in registers, ~2^-25 truncation per accumulation step), so the asserted bound is 3e-5 RMS."""
import pytest
import torch

import vits_oracle as O

pytestmark = pytest.mark.gpu
RMS_TOL = 3e-5
MAX_TOL = 3e-4


def _close(got, want):
    got, want = got.float().cpu(), want.float().cpu()
    assert got.shape == want.shape
    err = got - want
    rms = err.pow(2).mean().sqrt().item()
    assert rms <= RMS_TOL and err.abs().max().item() <= MAX_TOL, (rms, err.abs().max().item(), want.abs().max().item())
    ref = want.pow(2).mean().sqrt().item()
    assert rms <= 1e-4 * ref, f"relative RMS error {rms / ref} (signal RMS {ref})"


def _build(args):
    from tts_b200.hifigan import HifiganGenerator
    return HifiganGenerator(**args).eval()


def test_golden_v1_small(golden):
    g = golden("hifigan_v1_small")
    m = _build(g["args"])
    m.load_state_dict(g["state"])
    m.cuda()
    _close(m(g["x"].cuda()), g["y"])
    _close(m.inference(g["x"].cuda()), g["y_inference"])
    m.remove_weight_norm()
    _close(m(g["x"].cuda()), g["y"])


def test_golden_cond_resblock2(golden):
    g = golden("hifigan_cond_rb2_small")
    m = _build(g["args"])
    m.load_state_dict(g["state"])
    m.cuda()
    _close(m(g["x"].cuda(), g["g"].cuda()), g["y"])
    with pytest.raises(ValueError):
        m(g["x"].cuda())


def _oracle_kw(a):
    return dict(upsample_factors=a["upsample_factors"], upsample_kernel_sizes=a["upsample_kernel_sizes"],
                resblock_kernel_sizes=a["resblock_kernel_sizes"],
                resblock_dilation_sizes=a["resblock_dilation_sizes"], resblock_type=a["resblock_type"])


@pytest.mark.parametrize("b,t", [(2, 10), (1, 1), (3, 37)])
def test_full_width_vits_decoder_vs_oracle(b, t):
    torch.manual_seed(b * 100 + t)
    a = dict(in_channels=192, out_channels=1, resblock_type="1", resblock_dilation_sizes=[[1, 3, 5]] * 3,
             resblock_kernel_sizes=[3, 7, 11], upsample_kernel_sizes=[16, 16, 4, 4], upsample_initial_channel=512,
             upsample_factors=[8, 8, 2, 2], inference_padding=0, cond_channels=256, conv_pre_weight_norm=False,
             conv_post_weight_norm=False, conv_post_bias=False)
    m = _build(a)
    x, g = torch.randn(b, 192, t), torch.randn(b, 256, 1)
    want = O.hifigan_forward(m.state_dict(), x, g, **_oracle_kw(a))
    m.cuda()
    got = m(x.cuda(), g.cuda())
    assert got.shape == (b, 1, t * 256)
    _close(got, want)


def test_standalone_v1_cfg1_shape_vs_oracle():
    """BASELINE config 1 topology (80-band mel in, weight norm on); short T keeps the CPU oracle fast."""
    torch.manual_seed(7)
    a = dict(in_channels=80, out_channels=1, resblock_type="1", resblock_dilation_sizes=[[1, 3, 5]] * 3,
             resblock_kernel_sizes=[3, 7, 11], upsample_kernel_sizes=[16, 16, 4, 4], upsample_initial_channel=512,
             upsample_factors=[8, 8, 2, 2])
    m = _build(a)
    x = torch.randn(4, 80, 24)
    want = O.hifigan_forward(m.state_dict(), x, **_oracle_kw(a))
    m.cuda()
    _close(m(x.cuda()), want)


def test_odd_upsample_geometry_vs_oracle():
    """k - u odd => output length is not T*u; exercises the general polyphase tap range."""
    torch.manual_seed(3)
    a = dict(in_channels=20, out_channels=2, resblock_type="1", resblock_dilation_sizes=[[1, 2], [2, 6]],
             resblock_kernel_sizes=[3, 5], upsample_kernel_sizes=[7, 3], upsample_initial_channel=64,
             upsample_factors=[3, 2])
    m = _build(a)
    x = torch.randn(2, 20, 29)
    want = O.hifigan_forward(m.state_dict(), x, **_oracle_kw(a))
    m.cuda()
    _close(m(x.cuda()), want)
