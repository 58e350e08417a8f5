"""TEST INFRASTRUCTURE ONLY -- a CPU restatement of Tacotron.inference (TTS/tts/models/tacotron.py:218-271; the layers
in TTS/tts/layers/tacotron/tacotron.py) over a reference-format state dict, in torch on the CPU.

Each row runs on its own at its own length, i.e. the reference's inference(text[b:b+1, :x_lengths[b]]), which is what
the batched GPU drop-in computes, with the reference's stop rule: with t steps taken, stop once t > len / 4 and
(sigmoid(logit) > 0.6 or the attention weight at the last token > 0.6), or once t > max_decoder_steps.  Without
``draws`` the decoder prenet's dropout (when active) draws from torch's global generator in the reference's order; with
``draws`` ({"dropout": [B, S, 2, 256] bool}, layer 1 reading the first 128) a dropped unit is zero and a kept one
doubled -- the drop-in's mechanism.  ``dtype=torch.float64`` runs everything in double.  Also returns, per row, the stop
logits and the margins of both stop tests (the smallest |sigmoid - 0.6| and |alpha_last - 0.6| at the steps where the
rule is evaluated).
"""
import torch
import torch.nn.functional as F
from torch import nn

from tacotron2_oracle import _Attention, _sub


def _bn_conv(sd, p, x, k, act, dtype):
    o = F.conv1d(F.pad(x, [(k - 1) // 2, k // 2]), sd[p + "conv1d.weight"].to(dtype))
    o = F.batch_norm(o, sd[p + "bn.running_mean"].to(dtype), sd[p + "bn.running_var"].to(dtype),
                     sd[p + "bn.weight"].to(dtype), sd[p + "bn.bias"].to(dtype), False, 0.99, 1e-3)
    return act(o) if act else o


def cbhg(sd, p, x, K, dtype=torch.float32):
    """CBHG.forward (tacotron.py:162-188): x [1, Cin, T] -> [1, T, 256]."""
    y = torch.cat([_bn_conv(sd, f"{p}conv1d_banks.{k - 1}.", x, k, F.relu, dtype) for k in range(1, K + 1)], dim=1)
    y = _bn_conv(sd, p + "conv1d_projections.0.", y, 3, F.relu, dtype)
    y = _bn_conv(sd, p + "conv1d_projections.1.", y, 3, None, dtype)
    y = (y + x).transpose(1, 2)
    if p + "pre_highway.weight" in sd:
        y = F.linear(y, sd[p + "pre_highway.weight"].to(dtype))
    for i in range(4):
        h = F.relu(F.linear(y, sd[f"{p}highways.{i}.H.weight"].to(dtype), sd[f"{p}highways.{i}.H.bias"].to(dtype)))
        t = torch.sigmoid(F.linear(y, sd[f"{p}highways.{i}.T.weight"].to(dtype), sd[f"{p}highways.{i}.T.bias"].to(dtype)))
        y = h * t + y * (1.0 - t)
    gru = nn.GRU(128, 128, 1, batch_first=True, bidirectional=True, device="meta")
    gru.load_state_dict({k: v.to(dtype) for k, v in _sub(sd, p + "gru").items()}, assign=True)
    return gru(y)[0]


def encoder(sd, tokens, dtype=torch.float32):
    """embedding + Encoder (tacotron.py:210-229, eval) on one unpadded row [1, T] -> [1, T, 256]."""
    o = F.embedding(tokens, sd["embedding.weight"].to(dtype))
    for i in range(2):
        p = f"encoder.prenet.linear_layers.{i}.linear_layer."
        o = F.relu(F.linear(o, sd[p + "weight"].to(dtype), sd[p + "bias"].to(dtype)))
    return cbhg(sd, "encoder.cbhg.cbhg.", o.transpose(1, 2), 16, dtype)


def _prenet(sd, x, cfg, active, drop_row, dtype):
    for i in range(2):
        p = f"decoder.prenet.linear_layers.{i}."
        x = F.linear(x, sd[p + "linear_layer.weight"].to(dtype), sd[p + "linear_layer.bias"].to(dtype))
        if cfg["prenet_type"] == "bn":
            x = F.batch_norm(x, sd[p + "batch_normalization.running_mean"].to(dtype),
                             sd[p + "batch_normalization.running_var"].to(dtype),
                             sd[p + "batch_normalization.weight"].to(dtype), sd[p + "batch_normalization.bias"].to(dtype),
                             False, 0.1, 1e-5)
        x = F.relu(x)
        if cfg["prenet_dropout"]:
            if drop_row is not None:
                x = x * (drop_row[i][:x.shape[1]].to(x.device, dtype) * 2.0) if active else x
            else:
                x = F.dropout(x, p=0.5, training=active)
    return x


def _cell(sd, name, dtype):
    w = _sub(sd, name)
    cell = nn.GRUCell(w["weight_ih"].shape[1], 256, device="meta")
    cell.load_state_dict({k: v.to(dtype) for k, v in w.items()}, assign=True)
    return cell


def decode(sd, inputs, cfg, r, max_steps, drop=None, dtype=torch.float32):
    """Decoder.inference (tacotron.py:457-485) for one row: inputs [1, T, 256] -> (frames [r * steps, C], alignments
    [steps, T], stop values [steps], stop logits [steps], margins (stop, attention))."""
    c = cfg["decoder_output_dim"]
    active = bool(cfg["prenet_dropout"]) and bool(cfg["prenet_dropout_at_inference"])
    ms = cfg["memory_size"]
    z = dict(dtype=dtype, device=inputs.device)
    memory = torch.zeros(1, c * ms if ms > 0 else c, **z)
    arnn = _cell(sd, "decoder.attention_rnn", dtype)
    drnn = [_cell(sd, f"decoder.decoder_rnns.{i}", dtype) for i in range(2)]
    att = _Attention(sd, cfg, inputs, dtype)
    wd, bd = sd["decoder.project_to_decoder_in.weight"].to(dtype), sd["decoder.project_to_decoder_in.bias"].to(dtype)
    wp, bp = sd["decoder.proj_to_mel.weight"].to(dtype), sd["decoder.proj_to_mel.bias"].to(dtype)
    ws, bs = sd["decoder.stopnet.linear.weight"].to(dtype), sd["decoder.stopnet.linear.bias"].to(dtype)
    query = torch.zeros(1, 256, **z)
    hs = [torch.zeros(1, 256, **z) for _ in range(2)]
    context = torch.zeros(1, 256, **z)
    n_tok = inputs.shape[1]
    outs, aligns, stops, logits, t = [], [], [], [], 0
    m_stop, m_attn = float("inf"), float("inf")
    while True:
        pm = _prenet(sd, memory, cfg, active, None if drop is None else drop[t], dtype)
        query = arnn(torch.cat((pm, context), -1), query)
        context = att(query)
        x = F.linear(torch.cat((query, context), -1), wd, bd)
        for i in range(2):
            hs[i] = drnn[i](x, hs[i])
            x = hs[i] + x
        out = F.linear(x, wp, bp)
        logit = F.linear(torch.cat([x, out], -1), ws, bs)
        out = out[:, :r * c]
        stop = torch.sigmoid(logit.data)
        outs.append(out)
        aligns.append(att.w)
        stops.append(stop)
        logits.append(float(logit))
        t += 1
        if t > n_tok / 4:
            m_stop = min(m_stop, abs(float(stop) - 0.6))
            m_attn = min(m_attn, abs(float(att.w[:, -1]) - 0.6))
            if stop > 0.6 or att.w[:, -1].item() > 0.6:
                break
        if t > max_steps:
            break
        if ms > 0:   # _update_memory_input
            memory = torch.cat([out, memory[:, :(ms - r) * c]], -1) if ms > r else out[:, :ms * c]
        else:
            memory = out[:, c * (r - 1):]
    frames = torch.stack(outs).transpose(0, 1).contiguous().view(1, -1, c)[0]
    return frames, torch.cat(aligns, 0), torch.cat(stops, 0).flatten(), logits, (m_stop, m_attn)


def postnet(sd, dec, dtype=torch.float32):
    """last_linear(PostCBHG(decoder_outputs)) (tacotron.py:262-263) on one row [T, C] -> [T, out_channels]."""
    y = cbhg(sd, "postnet.cbhg.", dec.t().unsqueeze(0), 8, dtype)
    return F.linear(y, sd["last_linear.weight"].to(dtype), sd["last_linear.bias"].to(dtype))[0]


@torch.no_grad()
def inference(sd, text, x_lengths, cfg, *, r=None, max_steps=None, draws=None, dtype=torch.float32):
    """Tacotron.inference, each row at its own length.  Returns the reference's output dict padded to the longest row
    (zeros past each row) plus "model_outputs_len", "steps", "logits" and "margins" (per row: (stop, attention))."""
    r = cfg["r"] if r is None else r
    max_steps = cfg["max_decoder_steps"] if max_steps is None else max_steps
    rows = []
    for b in range(text.shape[0]):
        n = int(x_lengths[b])
        enc = encoder(sd, text[b:b + 1, :n], dtype)
        drop = None if draws is None else draws["dropout"][b]
        dec, al, st, lg, mg = decode(sd, enc, cfg, r, max_steps, drop, dtype)
        rows.append((dec, postnet(sd, dec, dtype), al, st, lg, mg))
    bsz, tt = text.shape[0], text.shape[1]
    t_dec = max(len(x[3]) for x in rows)
    c, oc = cfg["decoder_output_dim"], cfg["out_channels"]
    out = {"model_outputs": torch.zeros(bsz, t_dec * r, oc, dtype=dtype),
           "decoder_outputs": torch.zeros(bsz, t_dec * r, c, dtype=dtype),
           "alignments": torch.zeros(bsz, t_dec, tt, dtype=dtype),
           "stop_tokens": torch.zeros(bsz, t_dec, 1, dtype=dtype)}
    steps, logits, margins = [], [], []
    for b, (dec, mel, al, st, lg, mg) in enumerate(rows):
        s = len(st)
        out["decoder_outputs"][b, :s * r] = dec
        out["model_outputs"][b, :s * r] = mel
        out["alignments"][b, :s, :al.shape[1]] = al
        out["stop_tokens"][b, :s, 0] = st
        steps.append(s)
        logits.append(lg)
        margins.append(mg)
    out["model_outputs_len"] = torch.tensor(steps) * r
    out.update(steps=steps, logits=logits, margins=margins)
    return out


def seeded_weights(sd, seed, stop_bias=0.0, stop_gain=40.0):
    """Test weights on a reference-format state dict: BatchNorm statistics / affines drawn from a seeded generator (0 / 1
    would hide the folding); the stopnet weights scaled by ``stop_gain`` and its bias set to ``stop_bias``, so a test can
    place the stop decisions (a bias of -30 leaves them to the attention test)."""
    g = torch.Generator().manual_seed(seed)
    out = dict(sd)
    for k, v in sd.items():
        if ("batch_normalization" in k or ".bn." in k) and v.is_floating_point():
            if k.endswith("running_var"):
                out[k] = 0.5 + torch.rand(v.shape, generator=g)
            elif k.endswith("weight"):
                out[k] = 1.0 + 0.2 * torch.randn(v.shape, generator=g)
            else:
                out[k] = 0.1 * torch.randn(v.shape, generator=g)
    out["decoder.stopnet.linear.weight"] = sd["decoder.stopnet.linear.weight"] * stop_gain
    out["decoder.stopnet.linear.bias"] = torch.full_like(sd["decoder.stopnet.linear.bias"], stop_bias)
    return out
