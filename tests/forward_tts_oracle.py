"""TEST INFRASTRUCTURE ONLY -- CPU (PyTorch fp32) restatement of ``ForwardTTS.inference`` (TTS/tts/models/forward_tts.py:
672-714) over a reference-format state dict, the checker for tts_b200.forward_tts.  Pinned ``torch.equal`` to the
unmodified reference by tests/test_forward_tts_oracle_cpu.py.

``inference`` with ``x_lengths`` is the batched semantics of the drop-in: the per-row loop of single-utterance calls on
``x[b:b+1, :x_lengths[b]]``, zero-padded to the longest row."""
import math

import torch
import torch.nn.functional as F

import vits_oracle as O
from vits_oracle import sub


def fft_layer(sd, x, key_padding_mask, num_heads):
    """FFTransformer.forward in eval, tts/layers/generic/transformer.py:21-35: the attention output is added twice."""
    src = x.permute(2, 0, 1)
    c = src.shape[-1]
    src2, _ = F.multi_head_attention_forward(
        src, src, src, c, num_heads, sd["self_attn.in_proj_weight"], sd["self_attn.in_proj_bias"], None, None, False,
        0.1, sd["self_attn.out_proj.weight"], sd["self_attn.out_proj.bias"], training=False,
        key_padding_mask=key_padding_mask, need_weights=True, attn_mask=None)
    src = src + src2
    src = F.layer_norm(src + src2, (c,), sd["norm1.weight"], sd["norm1.bias"], 1e-5)
    src = src.permute(1, 2, 0)
    k = sd["conv1.weight"].shape[-1]
    src2 = F.conv1d(F.relu(F.conv1d(src, sd["conv1.weight"], sd["conv1.bias"], padding=(k - 1) // 2)),
                    sd["conv2.weight"], sd["conv2.bias"], padding=(k - 1) // 2)
    src = src + src2
    src = F.layer_norm(src.transpose(1, 2), (c,), sd["norm2.weight"], sd["norm2.bias"], 1e-5).transpose(1, 2)
    return src


def fft_block(sd, x, mask, num_heads):
    """FFTransformerBlock.forward, transformer.py:53-69 (mask [B, 1, T] or None)."""
    if mask is not None and mask.ndim == 3:
        mask = ~mask.squeeze(1).bool()
    n = len({k.split(".")[1] for k in sd if k.startswith("fft_layers.")})
    for i in range(n):
        x = fft_layer(sub(sd, f"fft_layers.{i}"), x, mask, num_heads)
    return x


def _predictor(sd, x, x_mask):
    return O.duration_predictor(sd, x, x_mask)


def inference_one(sd, x, args, length_scale=None, speaker_ids=None, d_vectors=None):
    """ForwardTTS.inference for one utterance x [1, T] (as the reference runs it); ``args`` is a ForwardTTSArgs."""
    if length_scale is None:
        length_scale = float(args.length_scale) if isinstance(args.length_scale, int) else args.length_scale
    g = speaker_ids if speaker_ids is not None else d_vectors
    x_lengths = torch.tensor(x.shape[1:2]).to(x.device)
    x_mask = torch.unsqueeze(O.sequence_mask(x_lengths, x.shape[1]), 1).to(x.dtype).float()
    # _forward_encoder (:399-415)
    if "emb_g.weight" in sd:
        g = F.embedding(g.type(torch.LongTensor), sd["emb_g.weight"])
    if g is not None:
        g = g.unsqueeze(-1)
    x_emb = F.embedding(x, sd["emb.weight"])
    o_en = fft_block(sub(sd, "encoder.encoder"), torch.transpose(x_emb, 1, -1), x_mask,
                     args.encoder_params["num_heads"]) * x_mask
    if g is not None:
        if "proj_g.weight" in sd:
            g = F.linear(g.view(g.shape[0], -1), sd["proj_g.weight"], sd["proj_g.bias"]).unsqueeze(-1)
        o_en = o_en + g
    o_dr_log = _predictor(sub(sd, "duration_predictor"), o_en.squeeze(), x_mask)
    # format_durations (:353-372)
    o_dr = (torch.exp(o_dr_log) - 1) * x_mask * length_scale
    o_dr[o_dr < 1] = 1.0
    o_dr = torch.round(o_dr).squeeze(1)
    y_lengths = o_dr.sum(1)
    o_pitch = o_energy = None
    if args.use_pitch:
        o_pitch = _predictor(sub(sd, "pitch_predictor"), o_en, x_mask)
        k = sd["pitch_emb.weight"].shape[-1]
        o_en = o_en + F.conv1d(o_pitch, sd["pitch_emb.weight"], sd["pitch_emb.bias"], padding=int((k - 1) / 2))
    if args.use_energy:
        o_energy = _predictor(sub(sd, "energy_predictor"), o_en, x_mask)
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
    o = fft_block(sub(sd, "decoder.decoder.transformer_block"), o_en_ex, None, args.decoder_params["num_heads"])
    o = o * y_mask
    o = F.conv1d(o, sd["decoder.decoder.postnet.weight"], sd["decoder.decoder.postnet.bias"]) * y_mask
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
