"""TEST INFRASTRUCTURE ONLY -- CPU (PyTorch fp32) restatement of ``ForwardTTS.inference`` (TTS/tts/models/forward_tts.py:
672-714) for SpeedySpeech, i.e. with encoder_type and decoder_type "residual_conv_bn" (TTS/tts/layers/generic/
res_conv_bn.py, feed_forward/encoder.py:41-73, feed_forward/decoder.py:125-160), over a reference-format state dict: the
checker for tts_b200.forward_tts.SpeedySpeech.  Pinned ``torch.equal`` to the unmodified reference by
tests/test_speedy_speech_oracle_cpu.py.  The text-side glue and the durations are tests/forward_tts_oracle.py's.

``inference`` with ``x_lengths`` is the batched semantics of the drop-in: the per-row loop of single-utterance calls on
``x[b:b+1, :x_lengths[b]]``, zero-padded to the longest row."""
import math

import torch
import torch.nn.functional as F

import forward_tts_oracle as FO
import vits_oracle as O
from vits_oracle import sub


def conv1d_bn(sd, x, dilation):
    """Conv1dBN.forward in eval, res_conv_bn.py:18-46: unpadded conv, ZeroPad2d((ps, pe, 0, 0)) on the output
    (ps = floor(d (k - 1) / 2)), ReLU, BatchNorm."""
    k = sd["conv1d.weight"].shape[-1]
    pad = dilation * (k - 1)
    o = F.conv1d(x, sd["conv1d.weight"], sd["conv1d.bias"], dilation=dilation)
    o = F.relu(F.pad(o, (pad // 2, pad - pad // 2)))
    return F.batch_norm(o, sd["norm.running_mean"], sd["norm.running_var"], sd["norm.weight"], sd["norm.bias"], False,
                        0.1, 1e-5)


def conv_bn_block(sd, x, dilation, num_conv_blocks):
    """Conv1dBNBlock.forward, res_conv_bn.py:76-83."""
    for j in range(num_conv_blocks):
        x = conv1d_bn(sub(sd, f"conv_bn_blocks.{j}"), x, dilation)
    return x


def res_conv_bn(sd, x, x_mask, params):
    """ResidualConv1dBNBlock.forward, res_conv_bn.py:129-137."""
    o = x * x_mask
    for i, d in enumerate(params["dilations"]):
        res = o
        o = conv_bn_block(sub(sd, f"res_blocks.{i}"), o, d, params["num_conv_blocks"])
        o = o + res
        o = o * x_mask
    return o


def encoder(sd, x, x_mask, params):
    """ResidualConv1dBNEncoder.forward, feed_forward/encoder.py:62-73 (x: the embedding)."""
    o = F.relu(F.conv1d(x, sd["prenet.0.weight"], sd["prenet.0.bias"])) * x_mask
    o = res_conv_bn(sub(sd, "res_conv_block"), o, x_mask, params)
    o = F.relu(F.conv1d(o + x, sd["postnet.0.weight"], sd["postnet.0.bias"]))
    o = F.batch_norm(o, sd["postnet.2.running_mean"], sd["postnet.2.running_var"], sd["postnet.2.weight"],
                     sd["postnet.2.bias"], False, 0.1, 1e-5)
    o = F.conv1d(o, sd["postnet.3.weight"], sd["postnet.3.bias"]) * x_mask
    return o * x_mask


def decoder(sd, x, x_mask, params):
    """ResidualConv1dBNDecoder.forward, feed_forward/decoder.py:154-160."""
    o = res_conv_bn(sub(sd, "res_conv_block"), x, x_mask, params)
    o = F.conv1d(o, sd["post_conv.weight"], sd["post_conv.bias"]) + x
    o = conv_bn_block(sub(sd, "postnet.0"), o, 1, 2)
    return F.conv1d(o, sd["postnet.1.weight"], sd["postnet.1.bias"]) * x_mask


def inference_one(sd, x, args, length_scale=None, speaker_ids=None, d_vectors=None):
    """ForwardTTS.inference for one utterance x [1, T] (as the reference runs it); ``args`` is a ForwardTTSArgs with the
    residual_conv_bn encoder and decoder."""
    if length_scale is None:
        length_scale = float(args.length_scale) if isinstance(args.length_scale, int) else args.length_scale
    g = speaker_ids if speaker_ids is not None else d_vectors
    x_lengths = torch.tensor(x.shape[1:2]).to(x.device)
    x_mask = torch.unsqueeze(O.sequence_mask(x_lengths, x.shape[1]), 1).to(x.dtype).float()
    # _forward_encoder (:399-415); Encoder.forward multiplies by x_mask once more (encoder.py:152)
    if "emb_g.weight" in sd:
        g = F.embedding(g.type(torch.LongTensor), sd["emb_g.weight"])
    if g is not None:
        g = g.unsqueeze(-1)
    x_emb = F.embedding(x, sd["emb.weight"])
    o_en = encoder(sub(sd, "encoder.encoder"), torch.transpose(x_emb, 1, -1), x_mask, args.encoder_params) * x_mask
    if g is not None:
        if "proj_g.weight" in sd:
            g = F.linear(g.view(g.shape[0], -1), sd["proj_g.weight"], sd["proj_g.bias"]).unsqueeze(-1)
        o_en = o_en + g
    o_dr_log = FO._predictor(sub(sd, "duration_predictor"), o_en.squeeze(), x_mask)
    # format_durations (:353-372)
    o_dr = (torch.exp(o_dr_log) - 1) * x_mask * length_scale
    o_dr[o_dr < 1] = 1.0
    o_dr = torch.round(o_dr).squeeze(1)
    y_lengths = o_dr.sum(1)
    o_pitch = o_energy = None
    if args.use_pitch:
        o_pitch = FO._predictor(sub(sd, "pitch_predictor"), o_en, x_mask)
        k = sd["pitch_emb.weight"].shape[-1]
        o_en = o_en + F.conv1d(o_pitch, sd["pitch_emb.weight"], sd["pitch_emb.bias"], padding=int((k - 1) / 2))
    if args.use_energy:
        o_energy = FO._predictor(sub(sd, "energy_predictor"), o_en, x_mask)
        k = sd["energy_emb.weight"].shape[-1]
        o_en = o_en + F.conv1d(o_energy, sd["energy_emb.weight"], sd["energy_emb.bias"], padding=int((k - 1) / 2))
    # _forward_decoder (:443-451)
    y_mask = torch.unsqueeze(O.sequence_mask(y_lengths, None), 1).to(o_en.dtype)
    attn_mask = torch.unsqueeze(x_mask, -1) * torch.unsqueeze(y_mask, 2)
    attn = O.generate_path(o_dr, attn_mask.squeeze(1)).to(o_dr.dtype)
    o_en_ex = torch.matmul(attn.squeeze(1).transpose(1, 2).to(o_en.dtype), o_en.transpose(1, 2)).transpose(1, 2)
    if "pos_encoder.pe" in sd:   # PositionalEncoding.forward, pos_encoding.py:38-69 (use_scale False)
        pe = sd["pos_encoder.pe"]
        o_en_ex = o_en_ex * math.sqrt(pe.shape[1])
        if pe.size(2) < o_en_ex.size(2):
            raise RuntimeError(f"Sequence is {o_en_ex.size(2)} but PositionalEncoding is"
                               f" limited to {pe.size(2)}. See max_len argument.")
        o_en_ex = o_en_ex + pe[:, :, : o_en_ex.size(2)] * y_mask
    o = decoder(sub(sd, "decoder.decoder"), o_en_ex, y_mask, args.decoder_params)
    return {"model_outputs": o.transpose(1, 2), "alignments": attn.transpose(1, 2), "pitch": o_pitch,
            "energy": o_energy, "durations_log": o_dr_log, "durations": o_dr, "y_lengths": y_lengths.long()}


def inference(sd, x, args, x_lengths=None, length_scale=None, speaker_ids=None, d_vectors=None):
    """The batched semantics: row b is ``inference_one(x[b:b+1, :x_lengths[b]])``, outputs zero-padded to the longest
    row ([B, T_de_max, C], [B, T_de_max, T], [B, 1, T], durations [B, T])."""
    b, t = x.shape
    if x_lengths is None:
        x_lengths = torch.full((b,), t, dtype=torch.int64)
    rows = []
    for i in range(b):
        n = int(x_lengths[i])
        rows.append(inference_one(sd, x[i: i + 1, :n], args, length_scale,
                                  None if speaker_ids is None else speaker_ids[i: i + 1],
                                  None if d_vectors is None else d_vectors[i: i + 1]))
    t_de = max(r["model_outputs"].shape[1] for r in rows)
    out = {"model_outputs": torch.zeros(b, t_de, rows[0]["model_outputs"].shape[2]),
           "alignments": torch.zeros(b, t_de, t), "durations_log": torch.zeros(b, 1, t), "durations": torch.zeros(b, t),
           "y_lengths": torch.cat([r["y_lengths"] for r in rows])}
    for k in ("pitch", "energy"):
        out[k] = None if rows[0][k] is None else torch.zeros(b, 1, t)
    for i, r in enumerate(rows):
        n, m = int(x_lengths[i]), r["model_outputs"].shape[1]
        out["model_outputs"][i, :m] = r["model_outputs"][0]
        out["alignments"][i, :m, :n] = r["alignments"][0]
        out["durations_log"][i, :, :n] = r["durations_log"][0]
        out["durations"][i, :n] = r["durations"][0]
        for k in ("pitch", "energy"):
            if r[k] is not None:
                out[k][i, :, :n] = r[k][0]
    return out
