"""The speaker encoder on the GPU against the CPU restatement (tests/encoder_oracle.py, pinned bit-exact to the reference
by tests/test_encoder_oracle_cpu.py), on the same inputs and seeded weights with randomised BatchNorm statistics."""
import numpy as np
import pytest
import torch

import encoder_oracle as EO
from tts_b200 import _lib
from tts_b200.encoder import ResNetSpeakerEncoder

pytestmark = pytest.mark.gpu

AUDIO = dict(fft_size=512, win_length=400, hop_length=160, sample_rate=16000, preemphasis=0.97, num_mels=64)
SR = 16000


def _rel(got, want):
    return float((got.double() - want.double()).norm() / want.double().norm())


def _rel_rms(got, want):
    return float((got.double() - want.double()).pow(2).mean().sqrt() / want.double().pow(2).mean().sqrt())


def _model(encoder_type="ASP", log_input=True, use_torch_spec=True, seed=1):
    m = ResNetSpeakerEncoder(encoder_type=encoder_type, log_input=log_input, use_torch_spec=use_torch_spec,
                             audio_config=AUDIO if use_torch_spec else None).eval()
    sd = EO.random_state(m.state_dict(), seed)
    m.load_state_dict(sd)
    return m.cuda(), sd


def _clip(n, seed):
    """A speech-like test signal: a few harmonics with a moving pitch under noise."""
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(n, dtype=torch.float64) / SR
    f0 = 110 + 60 * torch.rand(1, generator=g).item()
    ph = 2 * np.pi * torch.cumsum(f0 * (1 + 0.1 * torch.sin(2 * np.pi * 0.7 * t)), 0) / SR
    x = sum(torch.sin(k * ph) / k for k in range(1, 6)) * (0.5 + 0.5 * torch.sin(2 * np.pi * 2.1 * t) ** 2)
    return (0.3 * x + 0.02 * torch.randn(n, generator=g, dtype=torch.float64)).float()


def test_front_end_and_every_layer():
    m, sd = _model()
    x = torch.stack([_clip(40000, 1), _clip(40000, 2)]).unsqueeze(1)
    feats = EO.features(sd, x.clone(), AUDIO, True, True)
    layers = EO.trunk(sd, feats, (3, 4, 6, 3))
    got0 = m.forward_features(x.cuda(), 0).cpu()
    assert got0.shape == feats.shape and _rel_rms(got0, feats) <= 1e-5, _rel_rms(got0, feats)
    for s in range(1, 5):
        got = m.forward_features(x.cuda(), s).cpu()
        assert got.shape == layers[s - 1].shape, (s, got.shape)
        assert _rel_rms(got, layers[s - 1]) <= 1e-4, (s, _rel_rms(got, layers[s - 1]))


@pytest.mark.parametrize("encoder_type,log_input,use_torch_spec", [("ASP", True, True), ("SAP", False, True),
                                                                    ("ASP", False, False), ("SAP", True, False)])
def test_forward_variants(encoder_type, log_input, use_torch_spec):
    m, sd = _model(encoder_type, log_input, use_torch_spec, seed=4)
    if use_torch_spec:
        x = torch.stack([_clip(24000, 5), _clip(24000, 6), _clip(24000, 7)]).unsqueeze(1)
    else:
        x = torch.rand(3, 64, 180, generator=torch.Generator().manual_seed(2)) + (0.01 if log_input else -0.5)
    for l2 in (False, True):
        want = EO.forward(sd, x.clone(), AUDIO, encoder_type=encoder_type, log_input=log_input,
                          use_torch_spec=use_torch_spec, l2_norm=l2)
        got = m(x.cuda(), l2_norm=l2).cpu()
        assert got.shape == want.shape and _rel(got, want) <= 1e-4, (l2, _rel(got, want))


def test_compute_embedding_reference_defaults():
    """One 5 s clip at the reference's defaults: 10 windows of 250 frames (40000 samples)."""
    m, sd = _model()
    x = _clip(5 * SR, 11).unsqueeze(0)
    want = EO.compute_embedding(sd, x, AUDIO, encoder_type="ASP", log_input=True, use_torch_spec=True)
    got = m.compute_embedding(x.cuda()).cpu()
    assert got.shape == (1, 512) and _rel(got, want) <= 1e-4, _rel(got, want)
    per = m.compute_embedding(x.cuda(), return_mean=False).cpu()
    want_per = EO.compute_embedding(sd, x, AUDIO, return_mean=False, encoder_type="ASP", log_input=True,
                                    use_torch_spec=True)
    assert per.shape == (10, 512) and _rel(per, want_per) <= 1e-4


def test_compute_embedding_spectrogram_input():
    m, sd = _model("ASP", False, False, seed=8)
    x = torch.randn(1, 64, 300, generator=torch.Generator().manual_seed(4))
    want = EO.compute_embedding(sd, x, AUDIO, encoder_type="ASP", log_input=False, use_torch_spec=False)
    got = m.compute_embedding(x.cuda()).cpu()
    assert _rel(got, want) <= 1e-4, _rel(got, want)


def _dataset(n=64, seed=0):
    rng = np.random.default_rng(seed)
    lens = [int(rng.uniform(1.5, 8.0) * SR) for _ in range(n)]
    lens[:4] = [24000, 24000, 30000, 39999]    # short clips, two of one length (grouped by exact length)
    return [_clip(L, 100 + i) for i, L in enumerate(lens)]


def test_compute_embeddings_dataset_batch():
    m, sd = _model()
    clips = _dataset()
    got = m.compute_embeddings([c.cuda() for c in clips]).cpu()
    assert got.shape == (len(clips), 512)
    for i in range(0, len(clips), 1 if len(clips) <= 16 else 3):
        want = EO.compute_embedding(sd, clips[i].unsqueeze(0), AUDIO, encoder_type="ASP", log_input=True,
                                    use_torch_spec=True)
        assert _rel(got[i:i + 1], want) <= 1e-4, (i, _rel(got[i:i + 1], want))
    for i in (0, 2, 5, 17):
        one = m.compute_embedding(clips[i].cuda().unsqueeze(0)).cpu()
        assert _rel(got[i:i + 1], one) <= 1e-4, (i, _rel(got[i:i + 1], one))   # other batch, other tiling


def test_repeat_runs_bit_identical_and_nan_workspace():
    m, _ = _model()
    clips = [c.cuda() for c in _dataset(12, seed=3)]
    a = m.compute_embeddings(clips)
    b = m.compute_embeddings(clips)
    assert torch.equal(a, b)
    for buf in _lib._workspaces.values():
        buf.view(torch.uint8).fill_(0xFF)    # every float in the workspace reads as NaN
    c = m.compute_embeddings(clips)
    assert torch.equal(a, c)


def test_trunk_convs_dispatch_to_tensor_cores():
    """At the reference's defaults (one clip = 10 windows of 40000 samples) every SE-block conv, every downsample and
    both attention convs run on the 3xTF32 tensor-core kernels."""
    m, _ = _model()
    x = _clip(5 * SR, 12).unsqueeze(0).cuda()
    m.compute_embedding(x)
    torch.cuda.synchronize()
    with _lib.dispatch_log() as log:
        m.compute_embedding(x)
    torch.cuda.synchronize()
    assert _lib.lib().b200tts_debug_tc_error() == 0
    names = log.names
    n_blocks = 3 + 4 + 6 + 3
    # mel projection, stem conv, then per block conv1, conv2 (+ downsample), then attention x2 and fc
    assert len(names) == 2 + 2 * n_blocks + 3 + 3, names
    trunk = names[2:2 + 2 * n_blocks + 3 + 2]
    assert all(n in ("tc3", "tc3_grouped") for n in trunk), names


def test_zero_shot_d_vector_vits():
    """A d-vector VITS (d_vector_dim=512) fed the GPU embedding of a reference clip gives the durations and path of the
    oracle VITS fed the same embedding, and a waveform within the synthesis path's 1e-4 RMS gate."""
    from dataclasses import asdict

    import vits_oracle as O
    from tts_b200.vits import Vits, VitsArgs, VitsConfig

    enc, _ = _model()
    d = enc.compute_embedding(_clip(3 * SR, 21).unsqueeze(0).cuda())      # [1, 512], l2-normalised mean
    seed, b, t = 31, 1, 23
    cfg = VitsConfig(model_args=VitsArgs(use_d_vector_file=True, d_vector_dim=512, num_speakers=4))
    torch.manual_seed(seed)
    m = Vits(cfg).eval()
    gen = torch.Generator().manual_seed(seed)
    for _, p in m.named_parameters():
        if float(p.abs().sum()) == 0.0:
            p.data.copy_(torch.randn(p.shape, generator=gen) * 0.05)
    a = asdict(cfg.model_args)
    a["length_scale"] = 1.0
    tok = torch.randint(0, cfg.model_args.num_chars, (b, t))
    lens = torch.full((b,), t)
    sdp_noise = torch.randn(b, 2, t)
    store = {}

    def prior_noise(shape):
        store["n"] = torch.randn(shape, generator=torch.Generator().manual_seed(seed + 99))
        return store["n"]

    want = O.vits_inference(m.state_dict(), tok, lens, sdp_noise, prior_noise, args=a, d_vectors=d.cpu())
    m.cuda()
    got = m.inference(tok.cuda(), {"x_lengths": lens.cuda(), "d_vectors": d}, sdp_noise=sdp_noise,
                      prior_noise=lambda s: store["n"].cuda())
    assert torch.equal(got["durations"].cpu(), want["durations"])
    assert torch.equal(got["alignments"].cpu(), want["alignments"])
    assert got["model_outputs"].shape == want["model_outputs"].shape
    rms = float((got["model_outputs"].cpu() - want["model_outputs"]).pow(2).mean().sqrt())
    assert rms <= 1e-4, rms
