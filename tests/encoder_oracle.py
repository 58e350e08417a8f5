"""CPU restatement of the H/ASP speaker encoder (TTS/encoder/models/resnet.py:8-198 and base_encoder.py:12-96) as
functions of a state dict, in the same torch ops and order as the reference modules, so it is bit-exact against them
(tests/test_encoder_oracle_cpu.py pins that).  The GPU tests compare tts_b200.encoder against it.  It lives with the
tests, so the oracle module of the synthesis path is unchanged."""
import numpy as np
import torch
import torch.nn.functional as F


def _bn(sd, p, x):
    return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"], False,
                        0.0, 1e-5)


def front_end(sd, x, cfg):
    """x [B, T] waveform -> [B, n_mels, frames]: PreEmphasis, then torchaudio's MelSpectrogram (power 2, HTK, no norm)."""
    xp = F.pad(x.unsqueeze(1), (1, 0), "reflect")
    y = F.conv1d(xp, sd["torch_spec.0.filter"]).squeeze(1)
    spec = torch.stft(y, cfg["fft_size"], hop_length=cfg["hop_length"], win_length=cfg["win_length"],
                      window=sd["torch_spec.1.spectrogram.window"], center=True, pad_mode="reflect", normalized=False,
                      onesided=True, return_complex=True)
    spec = spec.abs().pow(2.0)
    return torch.matmul(spec.transpose(-1, -2), sd["torch_spec.1.mel_scale.fb"]).transpose(-1, -2)


def features(sd, x, cfg, log_input, use_torch_spec):
    """The instance-normed trunk input [B, n_mels, T] (resnet.py:164-171)."""
    if x.ndim == 3 and use_torch_spec:
        x = x.squeeze(1)
    if use_torch_spec:
        x = front_end(sd, x, cfg)
    if log_input:
        x = (x + 1e-6).log()
    return F.instance_norm(x, eps=1e-5)


def se_block(sd, p, x, stride):
    out = F.conv2d(x, sd[p + ".conv1.weight"], None, stride, 1)
    out = F.relu(out)
    out = _bn(sd, p + ".bn1", out)
    out = F.conv2d(out, sd[p + ".conv2.weight"], None, 1, 1)
    out = _bn(sd, p + ".bn2", out)
    b, c = out.shape[:2]
    y = F.adaptive_avg_pool2d(out, 1).view(b, c)
    y = F.relu(F.linear(y, sd[p + ".se.fc.0.weight"], sd[p + ".se.fc.0.bias"]))
    y = torch.sigmoid(F.linear(y, sd[p + ".se.fc.2.weight"], sd[p + ".se.fc.2.bias"])).view(b, c, 1, 1)
    out = out * y
    residual = x
    if (p + ".downsample.0.weight") in sd:
        residual = _bn(sd, p + ".downsample.1", F.conv2d(x, sd[p + ".downsample.0.weight"], None, stride))
    out += residual
    return F.relu(out)


def trunk(sd, x, layers):
    """[B, n_mels, T] -> the output of each of layer1..4 (list of four [B, C, H, T'] tensors)."""
    x = x.unsqueeze(1)
    x = _bn(sd, "bn1", F.relu(F.conv2d(x, sd["conv1.weight"], sd["conv1.bias"], 1, 1)))
    outs = []
    for s in range(4):
        for i in range(layers[s]):
            x = se_block(sd, f"layer{s + 1}.{i}", x, (2, 2) if (s > 0 and i == 0) else 1)
        outs.append(x)
    return outs


def head(sd, x, encoder_type, l2_norm):
    x = x.reshape(x.size()[0], -1, x.size()[-1])
    w = F.conv1d(x, sd["attention.0.weight"], sd["attention.0.bias"])
    w = _bn(sd, "attention.2", F.relu(w))
    w = torch.softmax(F.conv1d(w, sd["attention.3.weight"], sd["attention.3.bias"]), dim=2)
    if encoder_type == "SAP":
        x = torch.sum(x * w, dim=2)
    else:
        mu = torch.sum(x * w, dim=2)
        sg = torch.sqrt((torch.sum((x ** 2) * w, dim=2) - mu ** 2).clamp(min=1e-5))
        x = torch.cat((mu, sg), 1)
    x = F.linear(x.view(x.size()[0], -1), sd["fc.weight"], sd["fc.bias"])
    if l2_norm:
        x = F.normalize(x, p=2, dim=1)
    return x


def forward(sd, x, cfg, layers=(3, 4, 6, 3), encoder_type="ASP", log_input=False, use_torch_spec=False, l2_norm=False):
    """ResNetSpeakerEncoder.forward: x [B, 1, T] / [B, T] waveform or [B, n_mels, T] spectrogram -> [B, proj_dim]."""
    f = features(sd, x, cfg, log_input, use_torch_spec)
    return head(sd, trunk(sd, f, layers)[-1], encoder_type, l2_norm)


def window_offsets(max_len, num_frames, num_eval):
    """compute_embedding's window length and integer offsets (base_encoder.py:77-88)."""
    if max_len < num_frames:
        num_frames = max_len
    return num_frames, [int(o) for o in np.linspace(0, max_len - num_frames, num=num_eval)]


def compute_embedding(sd, x, cfg, num_frames=250, num_eval=10, return_mean=True, l2_norm=True, **kw):
    """BaseEncoder.compute_embedding (base_encoder.py:67-96): windows cut from x, run as one batch, averaged."""
    if kw.get("use_torch_spec"):
        num_frames = num_frames * cfg["hop_length"]
    nf, offsets = window_offsets(x.shape[1], num_frames, num_eval)
    frames = torch.cat([x[:, o:int(o + nf)] for o in offsets], dim=0)
    emb = forward(sd, frames, cfg, l2_norm=l2_norm, **kw)
    if return_mean:
        emb = torch.mean(emb, dim=0, keepdim=True)
    return emb


def random_state(state_dict, seed):
    """Seeded weights over a speaker-encoder state dict.  BatchNorm gets random running statistics and affine weights of
    both signs (the defaults -- mean 0, variance 1, weight 1 -- would hide where a BatchNorm sits relative to its ReLU);
    the front-end buffers (filter, window, filterbank) keep their values."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k, v in state_dict.items():
        if k.startswith("torch_spec") or not v.is_floating_point():
            out[k] = v.clone()
        elif k.endswith("running_var"):
            out[k] = torch.rand(v.shape, generator=g) + 0.5
        elif k.endswith("running_mean"):
            out[k] = torch.randn(v.shape, generator=g) * 0.3
        elif v.ndim >= 2:
            fan_in = int(np.prod(v.shape[1:]))
            out[k] = (torch.rand(v.shape, generator=g) * 2 - 1) * (3.0 / fan_in) ** 0.5
        elif ("bn" in k or "downsample.1" in k or "attention.2" in k) and k.endswith("weight"):
            out[k] = (torch.rand(v.shape, generator=g) * 2 - 1) * 1.5
        else:
            out[k] = torch.randn(v.shape, generator=g) * 0.1
    return out
