"""The speaker encoder without a GPU: the CPU restatement (tests/encoder_oracle.py) is pinned bit-exact to the
unmodified reference ``ResNetSpeakerEncoder`` -- live where the reference tree imports, through the results recorded
under tests/golden/reference/ elsewhere (regenerate with ``TTS_WRITE_GOLDEN=1 pytest tests/test_encoder_oracle_cpu.py``
where the reference is present) -- and the drop-in's surface (state-dict layout, checkpoint loading, window offsets,
setup_encoder_model, host-built front-end buffers) is checked against it."""
import importlib
import types

import numpy as np
import pytest
import torch

import encoder_oracle as EO
import ref_import
from ref_golden import Recorded, layout
from tts_b200.encoder import ResNetSpeakerEncoder, htk_mel_filterbank, setup_encoder_model

AUDIO = dict(fft_size=512, win_length=400, hop_length=160, sample_rate=16000, preemphasis=0.97, num_mels=64)


@pytest.fixture(scope="module")
def R():
    if not ref_import.available():
        return None
    ref_import.load_full()
    return importlib.import_module("TTS.encoder.models.resnet")


@pytest.fixture
def rec(request):
    r = Recorded(request.node.name)
    yield r
    r.save()


def _kw(encoder_type, log_input, use_torch_spec):
    return dict(encoder_type=encoder_type, log_input=log_input, use_torch_spec=use_torch_spec,
                audio_config=AUDIO if use_torch_spec else None)


def _ref_model(R, sd, **kw):
    m = R.ResNetSpeakerEncoder(**kw).eval()
    m.load_state_dict(sd)
    return m


@pytest.mark.parametrize("encoder_type", ["ASP", "SAP"])
@pytest.mark.parametrize("log_input", [True, False])
@pytest.mark.parametrize("use_torch_spec", [True, False])
def test_oracle_forward_equals_reference(R, rec, encoder_type, log_input, use_torch_spec):
    kw = _kw(encoder_type, log_input, use_torch_spec)
    sd = EO.random_state(ResNetSpeakerEncoder(**kw).state_dict(), 11)
    g = torch.Generator().manual_seed(3)
    if use_torch_spec:
        x = torch.randn(2, 1, 8000, generator=g) * 0.3
    else:
        x = torch.rand(2, 64, 40, generator=g) + (0.0 if log_input else -0.5)
    got = EO.forward(sd, x.clone(), AUDIO, l2_norm=True, encoder_type=encoder_type, log_input=log_input,
                     use_torch_spec=use_torch_spec)
    rec.check("emb", got, lambda: _ref_model(R, sd, **kw).inference(x.clone(), l2_norm=True))
    if use_torch_spec:
        ref_layers = lambda: _ref_model(R, sd, **kw).torch_spec(x.clone().squeeze(1))  # noqa: E731
        rec.check("mel", EO.front_end(sd, x.squeeze(1), AUDIO), ref_layers)


@pytest.mark.parametrize("n_samples", [60000, 30000, 12345])
def test_oracle_compute_embedding_equals_reference(R, rec, n_samples):
    """Long clip (overlapping windows), clip of about one window, clip shorter than a window (every window is the
    whole clip)."""
    kw = _kw("ASP", True, True)
    sd = EO.random_state(ResNetSpeakerEncoder(**kw).state_dict(), 5)
    x = torch.randn(1, n_samples, generator=torch.Generator().manual_seed(n_samples)) * 0.2
    got = EO.compute_embedding(sd, x, AUDIO, num_frames=100, num_eval=4, **{k: kw[k] for k in
                                                                         ("encoder_type", "log_input", "use_torch_spec")})
    rec.check("emb", got, lambda: _ref_model(R, sd, **kw).compute_embedding(x.clone(), num_frames=100, num_eval=4))


def test_oracle_compute_embedding_spectrogram_quirk(R, rec):
    """Spectrogram input: max_len is the mel axis, so every window is the whole [1, 64, T] input."""
    kw = _kw("ASP", False, False)
    sd = EO.random_state(ResNetSpeakerEncoder(**kw).state_dict(), 9)
    x = torch.randn(1, 64, 37, generator=torch.Generator().manual_seed(1))
    got = EO.compute_embedding(sd, x, AUDIO, num_eval=3, encoder_type="ASP", log_input=False, use_torch_spec=False)
    rec.check("emb", got, lambda: _ref_model(R, sd, **kw).compute_embedding(x.clone(), num_eval=3))


def test_window_plan_matches_reference_offsets():
    m = ResNetSpeakerEncoder(**_kw("ASP", True, True))
    for n in (40000, 40001, 80000, 123457, 39999, 16000, 400):
        nf, offs = m._window_plan(1, n, 250, 10)
        want_nf, want = EO.window_offsets(n, 250 * 160, 10)
        assert (nf, offs) == (want_nf, want)
        assert nf == min(n, 40000) and offs[0] == 0 and offs[-1] == n - nf
        if n < 40000:
            assert offs == [0] * 10


@pytest.mark.parametrize("use_torch_spec", [True, False])
def test_state_dict_layout_matches_reference(R, rec, use_torch_spec):
    kw = _kw("ASP", True, use_torch_spec)
    want = rec.value("layout", lambda: layout(R.ResNetSpeakerEncoder(**kw).state_dict()))
    got = layout(ResNetSpeakerEncoder(**kw).state_dict())
    assert [(k, s, d) for k, s, d, _ in got] == [(k, s, d) for k, s, d, _ in want]


def test_front_end_buffers_match_torchaudio(R, rec):
    """The host-built Hamming window and HTK filterbank equal the buffers torchaudio builds in the reference."""
    m = ResNetSpeakerEncoder(**_kw("ASP", True, True))
    mine = m.state_dict()
    for key in ("torch_spec.0.filter", "torch_spec.1.spectrogram.window", "torch_spec.1.mel_scale.fb"):
        rec.check(key, mine[key], lambda k=key: R.ResNetSpeakerEncoder(**_kw("ASP", True, True)).state_dict()[k])
    ta = pytest.importorskip("torchaudio")
    fb = ta.functional.melscale_fbanks(257, 0.0, 8000.0, 64, 16000, norm=None, mel_scale="htk")
    assert torch.equal(htk_mel_filterbank(257, 0.0, 8000.0, 64, 16000), fb)
    assert torch.equal(ta.transforms.Spectrogram(n_fft=512, win_length=400, window_fn=torch.hamming_window).window,
                       mine["torch_spec.1.spectrogram.window"])


def test_load_checkpoint_reference_format_strict(tmp_path):
    kw = _kw("ASP", True, True)
    sd = EO.random_state(ResNetSpeakerEncoder(**kw).state_dict(), 2)
    path = tmp_path / "encoder.pth"
    torch.save({"model": sd, "step": 7}, path)
    m = ResNetSpeakerEncoder(**kw)
    assert m.load_checkpoint(None, str(path), eval=True) is None
    assert not m.training
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k]), k
    m2 = ResNetSpeakerEncoder(**kw)
    assert m2.load_checkpoint(None, str(path), eval=False) == (None, 7)
    bad = dict(sd)
    bad.pop("fc.bias")
    torch.save({"model": bad, "step": 1}, path)
    with pytest.raises(RuntimeError):
        ResNetSpeakerEncoder(**kw).load_checkpoint(None, str(path), eval=True)


def test_setup_encoder_model():
    cfg = types.SimpleNamespace(model_params=dict(model_name="resnet", input_dim=64, proj_dim=512, log_input=True,
                                                  use_torch_spec=True), audio=AUDIO)
    m = setup_encoder_model(cfg)
    assert isinstance(m, ResNetSpeakerEncoder) and m.log_input and m.use_torch_spec and m.proj_dim == 512
    cfg.model_params["model_name"] = "LSTM"
    with pytest.raises(NotImplementedError):
        setup_encoder_model(cfg)
    cfg.model_params["model_name"] = "transformer"
    with pytest.raises(ValueError):
        setup_encoder_model(cfg)
    with pytest.raises(ValueError):
        ResNetSpeakerEncoder(encoder_type="XYZ")


def test_cpu_tensors_raise():
    if torch.cuda.is_available():
        pytest.skip("CPU-only check")
    m = ResNetSpeakerEncoder(**_kw("ASP", True, True))
    with pytest.raises(RuntimeError, match="no CPU path"):
        m(torch.zeros(1, 1, 8000))
    with pytest.raises(RuntimeError, match="no CPU path"):
        m.compute_embedding(torch.zeros(1, 8000))
    with pytest.raises(RuntimeError, match="no CPU path"):
        m.compute_embeddings([torch.zeros(8000)])
    assert np.isfinite(0.0)
