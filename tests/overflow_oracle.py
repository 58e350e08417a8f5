"""TEST INFRASTRUCTURE ONLY -- a CPU restatement of Overflow.inference and NeuralhmmTTS.inference
(TTS/tts/models/overflow.py:207-246, neuralhmm_tts.py; the layers in TTS/tts/layers/overflow/) over a reference-format
state dict, in torch on the CPU.

Each row runs on its own at its own length, i.e. the reference's inference(text[b:b+1, :x_lengths[b]]), which is what
the batched GPU drop-in computes.  Without ``draws`` the random numbers are taken from torch's global generator in the
reference's order (F.dropout, then Normal.sample, per frame), so a seeded call reproduces the reference; with ``draws``
({"noise": [B, F, C], "dropout": [B, F, L, P] bool}) the emission sample is mean + (std * temp) * noise and a dropped
prenet unit is zero, a kept one doubled -- the drop-in's mechanism.  ``dtype=torch.float64`` runs everything in double.
Also returns, per row, the smallest margin |quantile - threshold| met along the trajectory.
"""
import torch
import torch.distributions as tdist
import torch.nn.functional as F
from torch import nn

import glow_oracle as G


def _sub(sd, prefix):
    return {k[len(prefix) + 1:]: v for k, v in sd.items() if k.startswith(prefix + ".")}


def encoder(sd, tokens, cfg, dtype=torch.float32):
    """Encoder.inference (common_layers.py:70-92) on one unpadded row [1, T] -> states [1, T * spp, E]."""
    e = cfg["encoder_in_out_features"]
    spp = cfg["state_per_phone"]
    o = F.embedding(tokens, sd["encoder.emb.weight"].to(dtype)).transpose(1, 2)
    for i in range(cfg["encoder_n_convolutions"]):
        p = f"encoder.convolutions.{i}."
        o = F.conv1d(o, sd[p + "convolution1d.weight"].to(dtype), sd[p + "convolution1d.bias"].to(dtype), padding=2)
        o = F.batch_norm(o, sd[p + "batch_normalization.running_mean"].to(dtype),
                         sd[p + "batch_normalization.running_var"].to(dtype),
                         sd[p + "batch_normalization.weight"].to(dtype), sd[p + "batch_normalization.bias"].to(dtype),
                         False, 0.1, 1e-5)
        o = F.relu(o)
    o = o.transpose(1, 2)
    # built on the meta device so that no initialisation consumes the global generator the sampling draws from
    lstm = nn.LSTM(e, int(e / 2) * spp, num_layers=1, batch_first=True, bias=True, bidirectional=True, device="meta")
    lstm.load_state_dict({k: v.to(dtype) for k, v in _sub(sd, "encoder.lstm").items()}, assign=True)
    o, _ = lstm(o)
    b, t = tokens.shape
    return o.reshape(b, t * spp, e)


def _prenet(sd, x, cfg, active, drop_row, dtype):
    for i in range(cfg["prenet_n_layers"]):
        x = F.relu(F.linear(x, sd[f"neural_hmm.prenet.linear_layers.{i}.linear_layer.weight"].to(dtype)))
        if cfg["prenet_dropout"]:
            if drop_row is not None:
                x = x * (drop_row[i].to(dtype) * 2.0) if active else x
            else:
                x = F.dropout(x, p=0.5, training=active)
    return x


def _output_net(sd, h, z, cfg, dtype):
    """Outputnet.forward (common_layers.py:173-202) for one state."""
    x = torch.cat((h.unsqueeze(1), z), dim=2)
    p = "neural_hmm.output_net.parametermodel."
    for i in range(len(cfg["outputnet_size"])):
        x = F.relu(F.linear(x, sd[f"{p}layers.{i}.linear_layer.weight"].to(dtype),
                            sd[f"{p}layers.{i}.linear_layer.bias"].to(dtype)))
    x = F.linear(x, sd[p + "last_layer.weight"].to(dtype), sd[p + "last_layer.bias"].to(dtype))
    c = cfg["out_channels"]
    mean, std, tv = x[:, :, 0:c], x[:, :, c:2 * c], x[:, :, 2 * c:].squeeze(2)
    std = torch.clamp(F.softplus(std), min=cfg["std_floor"])
    return mean, std, tv


def sample(sd, inputs, n_states, cfg, temp, max_t, thr, noise=None, drop=None, dtype=torch.float32):
    """NeuralHMM.sample (neural_hmm.py:385-464) for one row: inputs [1, N, E] -> (x [T, C], states_travelled list,
    smallest |quantile - threshold|)."""
    c, ar = cfg["out_channels"], cfg["ar_order"]
    m = cfg["memory_rnn_dim"]
    cell = nn.LSTMCell(cfg["prenet_dim"], m, device="meta")
    cell.load_state_dict({k: v.to(dtype) for k, v in _sub(sd, "neural_hmm.memory_rnn").items()}, assign=True)
    active = bool(cfg["prenet_dropout_at_inference"])
    states, outs, t = [0], [], 0
    cur = 0
    prenet_input = sd["neural_hmm.go_tokens"].to(dtype).unsqueeze(0).expand(1, ar, c)
    h = torch.zeros(1, m, dtype=dtype, device=inputs.device)
    cc = torch.zeros(1, m, dtype=dtype, device=inputs.device)
    quantile = 1
    margin = float("inf")
    while True:
        mi = _prenet(sd, prenet_input.flatten(1).unsqueeze(0), cfg, active,
                     None if drop is None else drop[t], dtype)
        h, cc = cell(mi.squeeze(0), (h, cc))
        z_t = inputs[:, cur].unsqueeze(0)
        mean, std, tv = _output_net(sd, h, z_t, cfg, dtype)
        staying = torch.sigmoid(-tv.flatten())
        if temp > 0:
            if noise is not None:
                x_t = mean + (std * temp) * noise[t].to(dtype)
            else:
                x_t = tdist.normal.Normal(mean, std * temp).sample()
        else:
            x_t = mean
        prenet_input = torch.cat((prenet_input, x_t), dim=1)[:, 1:]
        outs.append(x_t.flatten())
        quantile *= staying
        margin = min(margin, abs(float(quantile) - thr))
        if quantile < thr:
            cur += 1
            quantile = 1
        states.append(cur)
        if cur == n_states or (max_t and t == max_t - 1):
            break
        t += 1
    return torch.stack(outs, dim=0), states, margin


@torch.no_grad()
def inference(sd, text, x_lengths, cfg, *, has_decoder, temp=None, max_t=None, thr=None, draws=None,
              dtype=torch.float32):
    """Overflow.inference / NeuralhmmTTS.inference, each row at its own length.  Returns the reference's output dict
    (without the plotting traces), plus "margins" (per row)."""
    temp = cfg["sampling_temp"] if temp is None else temp
    max_t = cfg["max_sampling_time"] if max_t is None else max_t
    thr = cfg["duration_threshold"] if thr is None else thr
    spp, c = cfg["state_per_phone"], cfg["out_channels"]
    rows, lens, aligns, margins = [], [], [], []
    for b in range(text.shape[0]):
        n = int(x_lengths[b])
        enc = encoder(sd, text[b:b + 1, :n], cfg, dtype)
        noise = None if draws is None or "noise" not in draws else draws["noise"][b]
        drop = None if draws is None or "dropout" not in draws else draws["dropout"][b]
        x, st, mg = sample(sd, enc, n * spp, cfg, temp, max_t, thr, noise, drop, dtype)
        rows.append(x)
        lens.append(x.shape[0])
        aligns.append(F.one_hot(torch.tensor(st)))
        margins.append(mg)
    hmm = nn.utils.rnn.pad_sequence(rows, batch_first=True)
    hmm_len = torch.tensor(lens, dtype=x_lengths.dtype)
    width = max(a.shape[1] for a in aligns)
    align = nn.utils.rnn.pad_sequence([F.pad(a, (0, width - a.shape[1])) for a in aligns], batch_first=True)
    mean, std = sd["mean"], sd["std"]
    if has_decoder:
        nsq = cfg["num_squeeze"]
        y_max = int(hmm_len.max() // nsq) * nsq
        y_len = torch.div(hmm_len, nsq, rounding_mode="floor") * nsq
        dsd = {k: v.to(dtype) if v.is_floating_point() else v for k, v in _sub(sd, "decoder.glow_decoder").items()}
        mels = []
        for b, row in enumerate(rows):   # each row through the decoder on its own, as the reference runs it
            n = int(y_len[b])
            y = row[:n].t().unsqueeze(0)
            out = G.decoder_reverse(dsd, y, torch.ones(1, 1, n, dtype=y.dtype), None,
                                    num_flow_blocks=cfg["num_flow_blocks_dec"], hidden=cfg["hidden_channels_dec"],
                                    kernel_size=cfg["kernel_size_dec"], dilation_rate=cfg["dilation_rate"],
                                    num_layers=cfg["num_block_layers"], num_splits=cfg["num_splits"], num_squeeze=nsq,
                                    sigmoid_scale=cfg["sigmoid_scale"])
            mels.append(F.pad(out, (0, y_max - n)))
        mel = torch.cat(mels, 0)
        mel = mel.transpose(1, 2).mul(std).add(mean)
        mel_len = y_len
    else:
        mel, mel_len = hmm.mul(std).add(mean), hmm_len
    return {"hmm_outputs": hmm, "hmm_outputs_len": hmm_len, "alignments": align, "model_outputs": mel,
            "model_outputs_len": mel_len, "margins": margins}


def seeded_weights(sd, seed):
    """Test weights on a reference-format state dict.  Randomly initialised weights are useless here: the flat-start
    output layer makes every state last the same number of frames, and BatchNorm statistics of 0 / 1 hide the folding.
    So the BatchNorm statistics / affines and the last output layer are drawn from a seeded generator, the transition
    row of the last layer is drawn ten times larger and the encoder-state columns of the first output layer thirty
    times larger: the encoder states are small (|z| ~ 0.05), and without that the transition logit hardly depends on
    the state, so every state of a row would again last the same number of frames."""
    g = torch.Generator().manual_seed(seed)
    out = dict(sd)
    m = sd["neural_hmm.memory_rnn.weight_hh"].shape[1]
    for k, v in sd.items():
        if "batch_normalization" in k and v.is_floating_point():
            if k.endswith("running_var"):
                out[k] = 0.5 + torch.rand(v.shape, generator=g)
            elif k.endswith("weight"):
                out[k] = 1.0 + 0.2 * torch.randn(v.shape, generator=g)
            else:
                out[k] = 0.1 * torch.randn(v.shape, generator=g)
        elif k.endswith("parametermodel.last_layer.weight"):
            w = torch.randn(v.shape, generator=g) * 0.3 / v.shape[1] ** 0.5
            w[-1] *= 10.0
            out[k] = w
        elif k.endswith("parametermodel.last_layer.bias"):
            b = 0.1 * torch.randn(v.shape, generator=g)
            b[-1] = -1.5 + 0.5 * torch.randn((), generator=g)
            out[k] = b
        elif k.endswith("parametermodel.layers.0.linear_layer.weight"):
            w = v.clone()
            w[:, m:] *= 30.0
            out[k] = w
    return out


def state_durations(alignments, frames):
    """Frames spent in each state of one row, from its [frames + 1, states] one-hot alignment."""
    st = alignments[:frames + 1].argmax(-1)
    return torch.bincount(st[:frames]).tolist()
