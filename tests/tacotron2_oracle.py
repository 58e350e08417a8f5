"""TEST INFRASTRUCTURE ONLY -- a CPU restatement of Tacotron2.inference (TTS/tts/models/tacotron2.py:238-300; the
layers in TTS/tts/layers/tacotron/) over a reference-format state dict, in torch on the CPU.

Each row runs on its own at its own length, i.e. the reference's inference(text[b:b+1, :x_lengths[b]]), which is what
the batched GPU drop-in computes; the reference's one-row stop rule applies (stop after step t >= 1 once
sigmoid(logit) > 0.5, or after max_decoder_steps steps, that step still emitted).  Without ``draws`` the prenet dropout
(when active) draws from torch's global generator in the reference's order; with ``draws`` ({"dropout": [B, S, 2, 256]
bool}) a dropped unit is zero and a kept one doubled -- the drop-in's mechanism.  ``dtype=torch.float64`` runs
everything in double.  Also returns, per row, the stop logits and the smallest |logit| met at the steps where the stop
rule is evaluated.
"""
import torch
import torch.nn.functional as F
from torch import nn


def _sub(sd, prefix):
    return {k[len(prefix) + 1:]: v for k, v in sd.items() if k.startswith(prefix + ".")}


def _conv_bn(sd, p, x, act, dtype):
    o = F.conv1d(x, sd[p + "convolution1d.weight"].to(dtype), sd[p + "convolution1d.bias"].to(dtype), padding=2)
    o = F.batch_norm(o, sd[p + "batch_normalization.running_mean"].to(dtype),
                     sd[p + "batch_normalization.running_var"].to(dtype), sd[p + "batch_normalization.weight"].to(dtype),
                     sd[p + "batch_normalization.bias"].to(dtype), False, 0.1, 1e-5)
    return act(o) if act else o


def encoder(sd, tokens, dtype=torch.float32):
    """embedding + Encoder.inference (tacotron2.py:105-112) on one unpadded row [1, T] -> [1, T, 512]."""
    o = F.embedding(tokens, sd["embedding.weight"].to(dtype)).transpose(1, 2)
    for i in range(3):
        o = _conv_bn(sd, f"encoder.convolutions.{i}.", o, F.relu, dtype)
    o = o.transpose(1, 2)
    lstm = nn.LSTM(512, 256, num_layers=1, batch_first=True, bias=True, bidirectional=True, device="meta")
    lstm.load_state_dict({k: v.to(dtype) for k, v in _sub(sd, "encoder.lstm").items()}, assign=True)
    o, _ = lstm(o)
    return o


def _prenet(sd, x, cfg, active, drop_row, dtype):
    for i in range(2):
        p = f"decoder.prenet.linear_layers.{i}."
        x = F.linear(x, sd[p + "linear_layer.weight"].to(dtype))
        if cfg["prenet_type"] == "bn":
            x = F.batch_norm(x, sd[p + "batch_normalization.running_mean"].to(dtype),
                             sd[p + "batch_normalization.running_var"].to(dtype),
                             sd[p + "batch_normalization.weight"].to(dtype), sd[p + "batch_normalization.bias"].to(dtype),
                             False, 0.1, 1e-5)
        x = F.relu(x)
        if cfg["prenet_dropout"]:
            if drop_row is not None:
                x = x * (drop_row[i].to(x.device, dtype) * 2.0) if active else x
            else:
                x = F.dropout(x, p=0.5, training=active)
    return x


class _Attention:
    """OriginalAttention / MonotonicDynamicConvolutionAttention forward (attentions.py) for one row, mask None."""

    def __init__(self, sd, cfg, inputs, dtype):
        self.p = {k: v.to(dtype) for k, v in _sub(sd, "decoder.attention").items()}
        self.cfg, self.inputs = cfg, inputs
        t = inputs.shape[1]
        self.dca = cfg["attention_type"] == "dynamic_convolution"
        self.w = torch.zeros([1, t], dtype=dtype, device=inputs.device)
        if self.dca:
            self.w[:, 0] = 1.0
        else:
            self.processed = F.linear(inputs, self.p["inputs_layer.linear_layer.weight"])
            if cfg["location_attn"]:
                self.cum = torch.zeros([1, t], dtype=dtype, device=inputs.device)

    def __call__(self, query):
        p = self.p
        if self.dca:
            prior = F.conv1d(F.pad(self.w.unsqueeze(1), (10, 0)), p["prior"].view(1, 1, -1))
            prior = torch.log(prior.clamp_min_(1e-6)).squeeze(1)
            g = F.linear(torch.tanh(F.linear(query, p["query_layer.weight"], p["query_layer.bias"])),
                         p["key_layer.weight"])
            dyn = F.conv1d(self.w.unsqueeze(0), g.view(-1, 1, 21), padding=10, groups=query.size(0))
            dyn = dyn.view(query.size(0), 8, -1).transpose(1, 2)
            stat = F.conv1d(self.w.unsqueeze(1), p["static_filter_conv.weight"], padding=10).transpose(1, 2)
            e = F.linear(torch.tanh(F.linear(stat, p["static_filter_layer.weight"]) +
                                    F.linear(dyn, p["dynamic_filter_layer.weight"], p["dynamic_filter_layer.bias"])),
                         p["v.weight"]).squeeze(-1) + prior
            a = F.softmax(e, dim=-1)
        else:
            pq = F.linear(query.unsqueeze(1), p["query_layer.linear_layer.weight"])
            vw, vb = p["v.linear_layer.weight"], p["v.linear_layer.bias"]
            if self.cfg["location_attn"]:
                cat = torch.cat((self.w.unsqueeze(1), self.cum.unsqueeze(1)), dim=1)
                pa = F.conv1d(cat, p["location_layer.location_conv1d.weight"], padding=15)
                pa = F.linear(pa.transpose(1, 2), p["location_layer.location_dense.linear_layer.weight"])
                e = F.linear(torch.tanh(pq + pa + self.processed), vw, vb).squeeze(-1)
            else:
                e = F.linear(torch.tanh(pq + self.processed), vw, vb).squeeze(-1)
            if self.cfg["attention_norm"] == "softmax":
                a = torch.softmax(e, dim=-1)
            else:
                a = torch.sigmoid(e) / torch.sigmoid(e).sum(dim=1, keepdim=True)
            if self.cfg["location_attn"]:
                self.cum += a
        self.w = a
        return torch.bmm(a.unsqueeze(1), self.inputs).squeeze(1)


def decode(sd, inputs, cfg, r, max_steps, drop=None, dtype=torch.float32):
    """Decoder.inference (tacotron2.py:329-367) for one row: inputs [1, T, 512] -> (frames [r * steps, C], alignments
    [steps, T], stop values [steps], stop logits [steps])."""
    c = cfg["out_channels"]
    active = bool(cfg["prenet_dropout"]) and bool(cfg["prenet_dropout_at_inference"])
    cells = []
    for n in ("attention_rnn", "decoder_rnn"):
        w = _sub(sd, "decoder." + n)
        cell = nn.LSTMCell(w["weight_ih"].shape[1], 1024, device="meta")
        cell.load_state_dict({k: v.to(dtype) for k, v in w.items()}, assign=True)
        cells.append(cell)
    att = _Attention(sd, cfg, inputs, dtype)
    wp, bp = sd["decoder.linear_projection.linear_layer.weight"].to(dtype), \
        sd["decoder.linear_projection.linear_layer.bias"].to(dtype)
    ws, bs = sd["decoder.stopnet.1.linear_layer.weight"].to(dtype), sd["decoder.stopnet.1.linear_layer.bias"].to(dtype)
    z = dict(dtype=dtype, device=inputs.device)
    memory = torch.zeros(1, c * r, **z)[:, c * (r - 1):]
    query, qc = torch.zeros(1, 1024, **z), torch.zeros(1, 1024, **z)
    dh, dc = torch.zeros(1, 1024, **z), torch.zeros(1, 1024, **z)
    context = torch.zeros(1, 512, **z)
    outs, aligns, stops, logits, t = [], [], [], [], 0
    while True:
        memory = _prenet(sd, memory, cfg, active, None if drop is None else drop[t], dtype)
        query, qc = cells[0](torch.cat((memory, context), -1), (query, qc))
        context = att(query)
        dh, dc = cells[1](torch.cat((query, context), -1), (dh, dc))
        out = F.linear(torch.cat((dh, context), dim=1), wp, bp)
        logit = F.linear(torch.cat((dh, out), dim=1), ws, bs)
        out = out[:, :r * c]
        stop = torch.sigmoid(logit.data)
        outs.append(out.squeeze(1))
        aligns.append(att.w)
        stops.append(stop)
        logits.append(float(logit))
        if stop > 0.5 and t > 0:
            break
        if len(outs) == max_steps:
            break
        memory = out[:, c * (r - 1):]
        t += 1
    frames = torch.stack(outs).transpose(0, 1).contiguous().view(1, -1, c)[0]
    return frames, torch.cat(aligns, 0), torch.cat(stops, 0).flatten(), logits


def postnet(sd, dec, dtype=torch.float32):
    """decoder_outputs + Postnet(decoder_outputs) (tacotron2.py:47-70) on one row [T, C] -> [T, C]."""
    x = dec.t().unsqueeze(0)
    o = x
    for i in range(5):
        o = _conv_bn(sd, f"postnet.convolutions.{i}.", o, torch.tanh if i < 4 else None, dtype)
    return (x + o)[0].t()


@torch.no_grad()
def inference(sd, text, x_lengths, cfg, *, r=None, max_steps=None, draws=None, dtype=torch.float32):
    """Tacotron2.inference, each row at its own length.  Returns the reference's output dict padded to the longest row
    (zeros past each row) plus "model_outputs_len", "steps", "logits" (per row) and "margins" (per row: the smallest
    |stop logit| at steps t >= 1)."""
    r = cfg["r"] if r is None else r
    max_steps = cfg["max_decoder_steps"] if max_steps is None else max_steps
    rows = []
    for b in range(text.shape[0]):
        n = int(x_lengths[b])
        enc = encoder(sd, text[b:b + 1, :n], dtype)
        drop = None if draws is None else draws["dropout"][b]
        dec, al, st, lg = decode(sd, enc, cfg, r, max_steps, drop, dtype)
        rows.append((dec, postnet(sd, dec, dtype), al, st, lg))
    bsz, tt = text.shape[0], text.shape[1]
    t_dec = max(len(x[3]) for x in rows)
    c = cfg["out_channels"]
    out = {"model_outputs": torch.zeros(bsz, t_dec * r, c, dtype=dtype),
           "decoder_outputs": torch.zeros(bsz, t_dec * r, c, dtype=dtype),
           "alignments": torch.zeros(bsz, t_dec, tt, dtype=dtype),
           "stop_tokens": torch.zeros(bsz, t_dec, 1, dtype=dtype)}
    steps, logits, margins = [], [], []
    for b, (dec, mel, al, st, lg) in enumerate(rows):
        s = len(st)
        out["decoder_outputs"][b, :s * r] = dec
        out["model_outputs"][b, :s * r] = mel
        out["alignments"][b, :s, :al.shape[1]] = al
        out["stop_tokens"][b, :s, 0] = st
        steps.append(s)
        logits.append(lg)
        margins.append(min((abs(v) for v in lg[1:]), default=float("inf")))
    out["model_outputs_len"] = torch.tensor(steps) * r
    out.update(steps=steps, logits=logits, margins=margins)
    return out


def seeded_weights(sd, seed, stop_bias=0.0, stop_gain=40.0):
    """Test weights on a reference-format state dict: BatchNorm statistics / affines drawn from a seeded generator (0 / 1
    would hide the folding); the stopnet weights scaled by ``stop_gain`` (at the default scale the stop logit hardly
    moves from its bias, so every row would stop at the same step) and its bias set to ``stop_bias``, so a test can
    place the stop decisions."""
    g = torch.Generator().manual_seed(seed)
    out = dict(sd)
    for k, v in sd.items():
        if "batch_normalization" in k and v.is_floating_point():
            if k.endswith("running_var"):
                out[k] = 0.5 + torch.rand(v.shape, generator=g)
            elif k.endswith("weight"):
                out[k] = 1.0 + 0.2 * torch.randn(v.shape, generator=g)
            else:
                out[k] = 0.1 * torch.randn(v.shape, generator=g)
    out["decoder.stopnet.1.linear_layer.weight"] = sd["decoder.stopnet.1.linear_layer.weight"] * stop_gain
    out["decoder.stopnet.1.linear_layer.bias"] = torch.full_like(sd["decoder.stopnet.1.linear_layer.bias"], stop_bias)
    return out
