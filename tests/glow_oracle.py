"""TEST INFRASTRUCTURE ONLY -- CPU (PyTorch fp32) restatement of ``GlowTTS.inference`` (TTS/tts/models/glow_tts.py:
341-374) over a reference-format state dict, the checker for tts_b200.glow_tts.  Built from vits_oracle's helpers;
pinned ``torch.equal`` to the unmodified reference by tests/test_glow_oracle_cpu.py."""
import math

import torch
import torch.nn.functional as F

import vits_oracle as O
from vits_oracle import conv_bias, conv_weight, sub


def layer_norm1(sd, x, eps=1e-4):
    """LayerNorm (type "1"), tts/layers/generic/normalization.py:23-28."""
    mean = torch.mean(x, 1, keepdim=True)
    variance = torch.mean((x - mean) ** 2, 1, keepdim=True)
    x = (x - mean) * torch.rsqrt(variance + eps)
    return x * sd["gamma"] + sd["beta"]


def prenet(sd, x, x_mask):
    """ResidualConv1dLayerNormBlock.forward, tts/layers/glow_tts/glow.py:55-67 (3 layers, kernel 5)."""
    x_res = x
    for i in range(3):
        x = F.conv1d(x * x_mask, sd[f"conv_layers.{i}.weight"], sd[f"conv_layers.{i}.bias"], padding=2)
        x = torch.relu(layer_norm1(sub(sd, f"norm_layers.{i}"), x * x_mask))
    x = x_res + F.conv1d(x, sd["proj.weight"], sd["proj.bias"])
    return x * x_mask


def transformer(sd, x, x_mask, *, num_layers, num_heads, kernel_size):
    """RelativePositionTransformer.forward, transformer.py:411-432, without a relative window, layer_norm_type "1"."""
    attn_mask = x_mask.unsqueeze(2) * x_mask.unsqueeze(-1)
    for i in range(num_layers):
        x = x * x_mask
        y = O.rel_attention(sub(sd, f"attn_layers.{i}"), x, attn_mask, num_heads=num_heads, window=None)
        x = layer_norm1(sub(sd, f"norm_layers_1.{i}"), x + y)
        y = O.ffn(sub(sd, f"ffn_layers.{i}"), x, x_mask, kernel_size)
        x = layer_norm1(sub(sd, f"norm_layers_2.{i}"), x + y)
    return x * x_mask


def encoder(sd, tokens, x_lengths, g=None, *, hidden, mean_only, use_prenet, num_layers, num_heads, kernel_size):
    """Encoder.forward, tts/layers/glow_tts/encoder.py:143-179 -> (o_mean, o_log_scale, logw, x_mask)."""
    x = F.embedding(tokens, sd["emb.weight"]) * math.sqrt(hidden)
    x = torch.transpose(x, 1, -1)
    x_mask = O.sequence_mask(x_lengths, x.size(2)).unsqueeze(1).to(x.dtype)
    if use_prenet:
        x = prenet(sub(sd, "prenet"), x, x_mask)
    x = transformer(sub(sd, "encoder"), x, x_mask, num_layers=num_layers, num_heads=num_heads, kernel_size=kernel_size)
    x_dp = torch.cat([x, g.expand(-1, -1, x.size(-1))], 1) if g is not None else x
    x_m = F.conv1d(x, sd["proj_m.weight"], sd["proj_m.bias"]) * x_mask
    x_logs = torch.zeros_like(x_m) if mean_only else F.conv1d(x, sd["proj_s.weight"], sd["proj_s.bias"]) * x_mask
    logw = O.duration_predictor(sub(sd, "duration_predictor"), x_dp, x_mask)
    return x_m, x_logs, logw, x_mask


def squeeze(x, x_mask, num_sqz):
    """decoder.py:8-28."""
    b, c, t = x.size()
    t = (t // num_sqz) * num_sqz
    x_sqz = x[:, :, :t].view(b, c, t // num_sqz, num_sqz).permute(0, 3, 1, 2).contiguous().view(b, c * num_sqz, t // num_sqz)
    x_mask = x_mask[:, :, num_sqz - 1::num_sqz]
    return x_sqz * x_mask, x_mask


def unsqueeze(x, x_mask, num_sqz):
    """decoder.py:31-47."""
    b, c, t = x.size()
    x_unsqz = x.view(b, num_sqz, c // num_sqz, t).permute(0, 2, 3, 1).contiguous().view(b, c // num_sqz, t * num_sqz)
    x_mask = x_mask.unsqueeze(-1).repeat(1, 1, 1, num_sqz).view(b, 1, t * num_sqz)
    return x_unsqz * x_mask, x_mask


def inv_conv_reverse(sd, x, x_mask, num_splits):
    """InvConvNear.forward(reverse=True), glow.py:102-137 (weight_inv if stored, else torch.inverse(weight.float()))."""
    b, c, t = x.size()
    x = x.view(b, 2, c // num_splits, num_splits // 2, t).permute(0, 1, 3, 2, 4).contiguous().view(b, num_splits,
                                                                                                 c // num_splits, t)
    weight = sd["weight_inv"] if "weight_inv" in sd else torch.inverse(sd["weight"].float()).to(sd["weight"].dtype)
    z = F.conv2d(x, weight.view(num_splits, num_splits, 1, 1))
    z = z.view(b, 2, num_splits // 2, c // num_splits, t).permute(0, 1, 3, 2, 4).contiguous().view(b, c, t)
    return z * x_mask


def coupling_reverse(sd, x, x_mask, g, *, hidden, kernel_size, dilation_rate, num_layers, sigmoid_scale):
    """CouplingBlock.forward(reverse=True), glow.py:201-230."""
    half = x.shape[1] // 2
    x_0, x_1 = x[:, :half], x[:, half:]
    h = F.conv1d(x_0, conv_weight(sd, "start"), conv_bias(sd, "start")) * x_mask
    h = O.wn_forward(sub(sd, "wn"), h, x_mask, g, hidden=hidden, kernel_size=kernel_size, dilation_rate=dilation_rate,
                     num_layers=num_layers)
    out = F.conv1d(h, sd["end.weight"], sd["end.bias"])
    t, s = out[:, :half], out[:, half:]
    if sigmoid_scale:
        s = torch.log(1e-6 + torch.sigmoid(s + 2))
    z_1 = (x_1 - t) * torch.exp(-s) * x_mask
    return torch.cat([x_0, z_1], 1)


def decoder_reverse(sd, x, x_mask, g, *, num_flow_blocks, hidden, kernel_size, dilation_rate, num_layers, num_splits,
                    num_squeeze, sigmoid_scale):
    """Decoder.forward(reverse=True), decoder.py:113-137."""
    if num_squeeze > 1:
        x, x_mask = squeeze(x, x_mask, num_squeeze)
    for n in reversed(range(num_flow_blocks)):
        x = coupling_reverse(sub(sd, f"flows.{3 * n + 2}"), x, x_mask, g, hidden=hidden, kernel_size=kernel_size,
                             dilation_rate=dilation_rate, num_layers=num_layers, sigmoid_scale=sigmoid_scale)
        x = inv_conv_reverse(sub(sd, f"flows.{3 * n + 1}"), x, x_mask, num_splits)
        an = sub(sd, f"flows.{3 * n}")
        x = (x - an["bias"]) * torch.exp(-an["logs"]) * x_mask        # ActNorm reverse, normalization.py:96-97
    if num_squeeze > 1:
        x, x_mask = unsqueeze(x, x_mask, num_squeeze)
    return x


def speaker_embedding(sd, speaker_ids=None, d_vectors=None):
    """_speaker_embedding, glow_tts.py:179-191: the l2-normalised [B, C, 1] speaker vector or None."""
    if speaker_ids is not None:
        if not speaker_ids.size():
            speaker_ids = speaker_ids.unsqueeze(0)
        return F.normalize(F.embedding(speaker_ids, sd["emb_g.weight"])).unsqueeze(-1)
    if d_vectors is not None:
        return F.normalize(d_vectors).unsqueeze(-1)
    return None


def inference(sd, x, x_lengths, cfg, *, speaker_ids=None, d_vectors=None, noise=None):
    """GlowTTS.inference, glow_tts.py:341-374; ``cfg`` is a GlowTTSConfig (or the reference's); ``noise`` replaces
    randn_like(y_mean) (needed when cfg.inference_noise_scale != 0)."""
    g = speaker_embedding(sd, speaker_ids, d_vectors)
    p = cfg.encoder_params
    o_mean, o_log_scale, o_dur_log, x_mask = encoder(
        sub(sd, "encoder"), x, x_lengths, g, hidden=cfg.hidden_channels_enc, mean_only=cfg.mean_only,
        use_prenet=cfg.use_encoder_prenet, num_layers=p["num_layers"], num_heads=p["num_heads"],
        kernel_size=p.get("kernel_size", 1))
    w = (torch.exp(o_dur_log) - 1) * x_mask * cfg.length_scale
    w_ceil = torch.clamp_min(torch.ceil(w), 1)
    y_lengths = torch.clamp_min(torch.sum(w_ceil, [1, 2]), 1).long()
    y_mask = O.sequence_mask(y_lengths, None).unsqueeze(1).to(x_mask.dtype)
    attn_mask = torch.unsqueeze(x_mask, -1) * torch.unsqueeze(y_mask, 2)
    attn = O.generate_path(w_ceil.squeeze(1), attn_mask.squeeze(1)).unsqueeze(1)
    y_mean = torch.matmul(attn.squeeze(1).transpose(1, 2), o_mean.transpose(1, 2)).transpose(1, 2)
    y_log_scale = torch.matmul(attn.squeeze(1).transpose(1, 2), o_log_scale.transpose(1, 2)).transpose(1, 2)
    o_attn_dur = torch.log(1 + torch.sum(attn, -1)) * x_mask
    if noise is None:
        noise = torch.randn_like(y_mean)
    z = (y_mean + torch.exp(y_log_scale) * noise * cfg.inference_noise_scale) * y_mask
    y = decoder_reverse(sub(sd, "decoder"), z, y_mask, g, num_flow_blocks=cfg.num_flow_blocks_dec,
                        hidden=cfg.hidden_channels_dec, kernel_size=cfg.kernel_size_dec,
                        dilation_rate=cfg.dilation_rate, num_layers=cfg.num_block_layers, num_splits=cfg.num_splits,
                        num_squeeze=cfg.num_squeeze, sigmoid_scale=cfg.sigmoid_scale)
    attn = attn.squeeze(1).permute(0, 2, 1)
    return {"model_outputs": y.transpose(1, 2), "logdet": None, "y_mean": y_mean.transpose(1, 2),
            "y_log_scale": y_log_scale.transpose(1, 2), "alignments": attn, "durations_log": o_dur_log.transpose(1, 2),
            "total_durations_log": o_attn_dur.transpose(1, 2), "durations": w_ceil, "y_lengths": y_lengths}
