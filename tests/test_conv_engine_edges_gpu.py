"""The conv engine (``launch_conv``) against float64 at the edges of its tiling and dispatch rules.

Every case is one ``FusedConv1d`` layer with a stated expected kernel family.  The expectation is derived from the
dispatch rules in ``try_launch_tc`` / ``launch_tiles`` / ``launch_conv`` / ``pack_rows`` (conv1d.cu); the comment on
each case names the rule it sits on, one or two values on either side:

  tensor cores (tc3 / tc3_grouped; tc16 / tc16_grouped for bf16 / fp16 with Cin % 16 == 0):
    rows >= 32 and Cin >= 8; Tq >= 128 (Tq = Tout, or ceil(Tout / stride) for transposed convs); 0 <= in_slope <= 1;
    no tanh; 16-byte aligned input rows; transposed convs only without residual / accumulate;
    rows_pad = round8(256 + (K - 1) * dil) <= 320 (plain mode)
  grouped mode: rows == 32 / 64 (G = 128 / rows tap groups), not transposed, Tq >= 256, (G - 1) * dil <= 15
  lean epilogue (inside tc3): no scale / post_div, interior 128-column half tiles, y / residual rows 16-byte aligned
  FMA tiles: co_tile 64 for rows >= 64 else 32; 8 input channels per stage for K >= 9 else 16; small_t for Tq <= 128;
    the 4-group split-K variant (KG = 4) for the plain epilogue with small_t, co_tile 64, <= 160 CTAs, >= 8 chunks
  row1: tanh, one output row, K 7, dil 1, pad 3, Tout % 4 == 0, 16-byte aligned rows

Each case is launched through ``b200tts_conv1d_forward_strided`` with the input inside a NaN-filled buffer (row pitch
round_up(T, 4): the tensor-core path stays eligible for odd T; NaN in the pitch columns, in spare channels past Cin and
in a batch row past the last) and the output inside NaN guards; then once more contiguously through
``FusedConv1d.__call__``, whose rows are not 16-byte aligned for T % 4 != 0, so that call is expected to run the FMA
kernel.  Every tensor-core case runs at tf32x3, f16x3, bf16 and fp16; every case also with ``tensor_cores=False``.

The reference is float64 on the device in the documented order ((conv(lrelu(x)) + bias) + res) * scale [+ y_old] /
post_div, or tests/lowp_reference.py for the 16-bit operand launches.  conv_check.py measures the error per (batch,
column) and per (batch, row) slice as well as over the whole tensor; FMA-kernel results are held to the error of
torch's fp32 CPU conv on the same inputs.  The measured maxima are printed at the end of the module (``-s``).
"""
import ctypes
from dataclasses import dataclass

import pytest
import torch

import conv_check as CC
from lowp_reference import lowp_conv1d
from test_bench_scale_gpu import LAYER_REL_TOL

pytestmark = pytest.mark.gpu

PRECS = ["tf32x3", "f16x3", "bf16", "fp16", "off"]   # off: tensor_cores=False
SPARE_CH = 2      # NaN channels past Cin in the strided input
GUARD = 64        # NaN floats before and after the output (keeps it 16-byte aligned)
NAN = float("nan")

# epilogues: residual, accumulate, scale, post_div, tanh (+ peak)
EPI = {
    "plain": {},
    "res": dict(res=True),                                   # lean epilogue with a residual
    "res_acc": dict(res=True, acc=True),                     # lean epilogue, residual + accumulate
    "scale": dict(scale=0.5),                                # general epilogue
    "div": dict(post_div=3.0),                               # general epilogue
    "mrf": dict(res=True, acc=True, post_div=3.0),           # ResBlock1 second conv + MRF mean: general epilogue
    "tanh": dict(tanh=True),                                 # conv_post, with the peak word
}


@dataclass(frozen=True)
class Case:
    name: str
    cin: int
    cout: int
    k: int
    family: str          # strided launch at tf32x3: "tc3", "tc3_grouped", "fma" or "row1"
    dil: int = 1
    pad: int = -1        # -1: "same", dil * (k - 1) // 2
    b: int = 2
    t: int = 300
    slope: float = 0.1
    epi: str = "plain"
    stride: int = 0      # > 0: transposed conv, weight [cin, cout, k]

    @property
    def padding(self):
        return self.dil * (self.k - 1) // 2 if self.pad < 0 else self.pad

    @property
    def rows(self):
        return self.cout * max(1, self.stride)


C = Case


CASES = [
    # ---- Tq >= 128 (rows 80, plain mode)
    C("tq124", 16, 80, 3, "fma", t=124),                      # Tq 124 < 128
    C("tq127_valid", 16, 80, 3, "fma", t=129, pad=0),         # Tq 127, Tout < T
    C("tq128", 16, 80, 3, "tc3", t=128),                      # Tq 128: first eligible
    C("tq128_valid", 16, 80, 3, "tc3", t=130, pad=0),
    C("tq129", 16, 80, 3, "tc3", t=129),                      # odd Tout: scalar stores, general epilogue
    C("tq131", 16, 80, 3, "tc3", t=131),
    # ---- grouped mode needs Tq >= 256 (rows 64: G = 2), and its 240-column tiles
    C("g_tq252", 64, 64, 3, "tc3", t=252),                    # Tq < 256: plain mode
    C("g_tq255", 64, 64, 3, "tc3", t=255),
    C("g_tq256", 64, 64, 3, "tc3_grouped", t=256),            # Tq >= 256: grouped
    C("g_tq257", 64, 64, 3, "tc3_grouped", t=257),
    C("g_tq240", 64, 64, 3, "tc3", t=240),                    # one grouped tile's width, but Tq < 256
    C("g_tq241", 32, 32, 3, "tc3", t=241),
    C("g_tq480", 64, 64, 3, "tc3_grouped", t=480),            # two 240-column tiles exactly
    C("g_tq481", 32, 32, 5, "tc3_grouped", t=481),            # a third tile with one column
    # ---- lean vs general epilogue on half tiles (rows 96, residual + accumulate)
    C("half380", 32, 96, 5, "tc3", t=380, epi="res_acc"),     # third half [256, 384) not interior: general
    C("half383", 32, 96, 5, "tc3", t=383, epi="res_acc"),     # y rows not 16-byte aligned: general everywhere
    C("half384", 32, 96, 5, "tc3", t=384, epi="res_acc"),     # three interior halves: lean
    C("half385", 32, 96, 5, "tc3", t=385, epi="res_acc"),
    C("half388", 32, 96, 5, "tc3", t=388, epi="res_acc"),     # three lean halves, a 4-column general half
    # ---- rows: FMA below 32 (co_tile 32), grouped at 32 / 64, partial 128-row tiles otherwise
    C("rows16", 16, 16, 3, "fma"),
    C("rows31", 16, 31, 3, "fma"),
    C("rows32", 16, 32, 3, "tc3_grouped"),
    C("rows33", 16, 33, 3, "tc3"),
    C("rows64", 16, 64, 3, "tc3_grouped"),
    C("rows80", 16, 80, 3, "tc3"),
    C("rows96", 16, 96, 3, "tc3"),
    C("rows127", 16, 127, 3, "tc3"),
    C("rows128", 16, 128, 3, "tc3"),
    C("rows129", 16, 129, 3, "tc3"),                          # second row tile with one row
    C("rows150", 16, 150, 3, "tc3"),
    C("rows192", 16, 192, 3, "tc3"),
    C("rows300", 16, 300, 3, "tc3"),
    C("rows384", 16, 384, 3, "tc3"),
    C("rows513", 16, 513, 3, "tc3"),
    # ---- Cin: FMA below 8; partial 8- / 16-channel chunks (16-bit requests with Cin % 16 != 0 run 3xTF32)
    C("cin1", 1, 80, 3, "fma"),
    C("cin7", 7, 80, 3, "fma"),
    C("cin8", 8, 80, 3, "tc3"),
    C("cin12", 12, 80, 3, "tc3"),
    C("cin13", 13, 80, 3, "tc3"),
    C("cin16", 16, 80, 3, "tc3"),
    C("cin80", 80, 80, 3, "tc3"),
    C("cin150", 150, 80, 3, "tc3"),
    C("cin200", 200, 80, 3, "tc3"),
    C("cin513", 513, 80, 3, "tc3"),
    C("cin13_g64", 13, 64, 3, "tc3_grouped"),                 # Cin tail in grouped mode
    C("cin8_g32", 8, 32, 5, "tc3_grouped"),
    # ---- K / dil / pad: K = 1, even K, "valid" (Tout < T) and over-padded (Tout > T)
    C("k1", 32, 80, 1, "tc3"),
    C("k2_valid", 32, 80, 2, "tc3", pad=0),
    C("k2_pad1", 32, 80, 2, "tc3", pad=1),
    C("k4_pad2", 24, 80, 4, "tc3", pad=2),
    C("k5_d2", 32, 80, 5, "tc3", dil=2),
    C("k7_d3_valid", 24, 80, 7, "tc3", dil=3, pad=0),
    C("k11_over", 32, 80, 11, "tc3", pad=10, t=301),
    C("k3_over", 32, 80, 3, "tc3", pad=3),
    C("g64_k1", 32, 64, 1, "tc3_grouped"),                    # grouped: K not a multiple of G (zero-padded taps)
    C("g64_k2", 32, 64, 2, "tc3_grouped", pad=0),
    C("g64_k5", 32, 64, 5, "tc3_grouped", t=301),
    C("g64_k7_valid", 32, 64, 7, "tc3_grouped", dil=2, pad=0, t=303),
    C("g64_k11_d5", 64, 64, 11, "tc3_grouped", dil=5),
    C("g32_k1", 32, 32, 1, "tc3_grouped"),
    C("g32_k7_d5", 32, 32, 7, "tc3_grouped", dil=5),          # (G-1)*dil = 15, K 7 = 2 tap blocks of 4
    C("g32_k11", 32, 32, 11, "tc3_grouped", t=299),
    C("g32_k3_over", 32, 32, 3, "tc3_grouped", pad=5),
    # ---- grouped-mode dilation limit (G - 1) * dil <= 15
    C("g64_d15", 64, 64, 3, "tc3_grouped", dil=15),
    C("g64_d16", 64, 64, 3, "tc3", dil=16),
    C("g32_d5", 32, 32, 3, "tc3_grouped", dil=5),
    C("g32_d6", 32, 32, 3, "tc3", dil=6),
    # ---- plain-window limit rows_pad = round8(256 + (K - 1) * dil) <= 320
    C("win_k3_d32", 32, 80, 3, "tc3", dil=32),                # 320
    C("win_k3_d33", 32, 80, 3, "fma", dil=33),                # 328
    C("win_k11_d6", 32, 80, 11, "tc3", dil=6),                # 320
    C("win_k11_d7", 32, 80, 11, "fma", dil=7),                # 328
    C("win_g64_k3_d33", 64, 64, 3, "fma", dil=33),            # neither grouped ((G-1)*dil > 15) nor plain
    # ---- epilogues (rows 96): lean with residual / accumulate, general with scale / post_div; in_slope in [0, 1]
    C("epi_res", 32, 96, 3, "tc3", epi="res"),
    C("epi_res_acc", 32, 96, 3, "tc3", epi="res_acc"),
    C("epi_scale", 32, 96, 3, "tc3", epi="scale"),
    C("epi_div", 32, 96, 3, "tc3", epi="div"),
    C("epi_mrf", 32, 96, 3, "tc3", epi="mrf"),
    C("epi_mrf_t301", 32, 96, 3, "tc3", epi="mrf", t=301),    # general epilogue, scalar stores
    C("epi_mrf_g64", 64, 64, 3, "tc3_grouped", epi="mrf", t=301),
    C("epi_scale_g32", 32, 32, 7, "tc3_grouped", epi="scale"),
    C("slope1", 32, 96, 3, "tc3", slope=1.0),
    C("slope0", 32, 96, 3, "tc3", slope=0.0),
    C("slope0.2", 32, 96, 3, "tc3", slope=0.2),
    C("slope1.5", 32, 96, 3, "fma", slope=1.5),               # outside [0, 1]: the producers' max(x, slope * x) is wrong
    C("slope1.5_g64", 32, 64, 3, "fma", slope=1.5),
    # ---- tanh: row1 for one row / K 7 / pad 3 / Tout % 4 == 0, else the FMA tanh + a separate peak pass
    C("tanh_row1", 32, 1, 7, "row1", t=256, epi="tanh"),
    C("tanh_row1_t258", 32, 1, 7, "fma", t=258, epi="tanh"),
    C("tanh_row1_t255", 32, 1, 7, "fma", t=255, epi="tanh"),
    C("tanh_cout4", 32, 4, 7, "fma", t=256, epi="tanh"),
    C("tanh_rows64", 64, 64, 3, "fma", epi="tanh"),           # tanh never runs on the tensor cores
    # ---- transposed: stride s, Kt in {s, 2s, 2s+1, 16}, padding in {0, (Kt-s)//2, s//2 + s%2}; rows = Cout * s
    C("tr_s2_k4_p1", 32, 16, 4, "tc3", stride=2, pad=1, t=150),           # rows 32
    C("tr_s2_k2_p0", 32, 8, 2, "fma", stride=2, pad=0, t=150),            # rows 16 < 32
    C("tr_s2_k5_p1_tq127", 32, 16, 5, "fma", stride=2, pad=1, t=126),     # Tout 253: Tq 127
    C("tr_s2_k5_p1_tq128", 32, 16, 5, "tc3", stride=2, pad=1, t=127),     # Tout 255: Tq 128
    C("tr_s3_k7_p2", 24, 16, 7, "tc3", stride=3, pad=2, t=151),           # rows 48, Cin tail
    C("tr_s3_k3_p2", 16, 32, 3, "tc3", stride=3, pad=2, t=150),           # rows 96
    C("tr_s4_k8_p2", 64, 32, 8, "tc3", stride=4, pad=2, t=150),           # rows 128
    C("tr_s4_k16_p6", 64, 16, 16, "tc3", stride=4, pad=6, t=149),         # rows 64: transposed never grouped
    C("tr_s4_k9_p0", 16, 8, 9, "tc3", stride=4, pad=0, t=150),
    C("tr_s5_k11_p3", 13, 8, 11, "tc3", stride=5, pad=3, t=150),          # rows 40
    C("tr_s5_k5_p0", 16, 4, 5, "fma", stride=5, pad=0, t=150),            # rows 20
    C("tr_s8_k16_p4", 128, 64, 16, "tc3", stride=8, pad=4, t=150),        # rows 512
    C("tr_s8_k8_p4", 32, 4, 8, "tc3", stride=8, pad=4, t=150),            # rows 32
    C("tr_s8_k17_p0", 16, 2, 17, "fma", stride=8, pad=0, t=150),          # rows 16
    C("tr_res", 32, 32, 4, "fma", stride=2, pad=1, t=150, epi="res"),     # residual: not persistent-eligible
    # ---- FMA tile variants (all log fma)
    C("fma_cic8_co32", 16, 16, 11, "fma", dil=2),             # K >= 9: 8 channels per stage; rows < 64: co_tile 32
    C("fma_cic8_co32_k9", 24, 31, 9, "fma", t=301),
    C("fma_cic16_co64", 7, 80, 3, "fma", t=301),              # Cin < 8: FMA; rows >= 64: co_tile 64
    C("fma_small_t_co64", 7, 80, 5, "fma", t=100),            # Tq <= 128: small_t tiles
    C("fma_small_t_co32", 24, 20, 3, "fma", t=99),
    C("fma_kg4_b8", 200, 192, 3, "fma", t=64, b=8),           # KG = 4: 24 CTAs, 13 channel chunks (not a multiple of 4)
    C("fma_kg4_b32", 200, 192, 3, "fma", t=64, b=32),         # 96 CTAs
    C("fma_kg1_b64", 200, 192, 3, "fma", t=64, b=64),         # 192 CTAs > 160: no split
    C("small_t_tq128", 150, 64, 3, "tc3", t=130, pad=0, b=4),  # Tq 128: tensor cores; off: KG = 4 over 2 column tiles
    # ---- many tiles per CTA at an edge shape: 300 x 2 partial tiles > 132 SMs
    C("many_tiles", 150, 150, 3, "tc3", t=129, b=300),
    # ---- named model layers
    C("overflow_decoder_in_layer", 150, 300, 5, "tc3", t=257),          # hidden 150, gate rows 300 (plain epilogue)
    C("fastpitch_ffn2", 1536, 384, 3, "tc3", t=200),                    # 384 channels: 3 row tiles
    C("fastpitch_postnet_proj", 384, 80, 1, "tc3", t=203),              # mel projection 384 -> 80
    C("posterior_encoder_pre", 513, 192, 1, "tc3", t=301),              # 513 linear-spectrogram inputs
    C("speaker_encoder_c2", 192, 64, 3, "tc3_grouped", t=301),          # Cin = 3C, C = 64
    C("speaker_encoder_c1_k2", 384, 128, 2, "tc3", pad=1, t=300),       # Cin = 6C, K 2 pad 1: Tout = T + 1
    C("hifigan_v2_last_resblock", 16, 16, 11, "fma", dil=5, t=2048, epi="mrf"),   # 16 channels: rows < 32
    C("hifigan_v2_last_upsampler", 32, 16, 4, "tc3", stride=2, pad=1, t=1024),    # 32 -> 16: rows 32
    C("hifigan_v2_conv_post", 16, 1, 7, "row1", t=2048, epi="tanh"),
    C("vits_text_encoder_ffn2", 768, 192, 3, "fma", t=64, b=32),        # T 64 < 128; KG = 4 (96 CTAs)
]
assert len({c.name for c in CASES}) == len(CASES)


def expected_family(case, prec, strided=True):
    """Kernel family a launch of `case` logs.  tensor_cores=False: FMA (row1 is not a tensor-core kernel); a contiguous
    input whose rows are not 16-byte aligned (T % 4 != 0): FMA; bf16 / fp16 with Cin % 16 == 0: the 16-bit tensor-core
    families; f16x3 (and 16-bit requests with Cin % 16 != 0) log as 3xTF32."""
    fam = case.family
    if fam == "row1":
        return "row1" if strided or case.t % 4 == 0 else "fma"
    if prec == "off" or fam == "fma" or (not strided and case.t % 4):
        return "fma"
    if prec in ("bf16", "fp16") and case.cin % 16 == 0:
        return fam.replace("tc3", "tc16")
    return fam


# ----------------------------------------------------------------------------- inputs, references, launches
_INPUTS, _WANT64, _CPU32, _RUNS = {}, {}, {}, {}
_STATS = {}


def _inputs(case):
    v = _INPUTS.get(case.name)
    if v is None:
        g = torch.Generator().manual_seed(sum(map(ord, case.name)))
        x = torch.randn(case.b, case.cin, case.t, generator=g)
        if case.stride:
            w = torch.randn(case.cin, case.cout, case.k, generator=g) / (case.cin * case.k / case.stride) ** 0.5
        else:
            w = torch.randn(case.cout, case.cin, case.k, generator=g) / (case.cin * case.k) ** 0.5
        bias = torch.randn(case.cout, generator=g) * 0.1
        tout = _conv_ref(case, x, w, bias, torch.float32).shape[-1]
        e = EPI[case.epi]
        res = torch.randn(case.b, case.cout, tout, generator=g) if e.get("res") else None
        y_old = torch.randn(case.b, case.cout, tout, generator=g) if e.get("acc") else None
        v = _INPUTS[case.name] = dict(x=x, w=w, bias=bias, res=res, y_old=y_old)
    return v


def _conv_ref(case, x, w, bias, dtype):
    return CC.conv(x, w, bias, dilation=case.dil, padding=case.padding, transposed=bool(case.stride),
                   stride=max(1, case.stride), in_slope=case.slope, dtype=dtype)


def _epi_ref(case, c, inp):
    e = EPI[case.epi]
    dev = c.device
    return CC.epilogue(c, residual=None if inp["res"] is None else inp["res"].to(dev),
                       scale=e.get("scale", 1.0), y_old=None if inp["y_old"] is None else inp["y_old"].to(dev),
                       post_div=e.get("post_div", 1.0), tanh=e.get("tanh", False))


def _want(case, family, prec):
    """float64 reference on the device; the 16-bit operand families against lowp_reference"""
    inp = _inputs(case)
    key = (case.name, prec if family.startswith("tc16") else "f64")
    if key not in _WANT64:
        x, w, bias = (inp[k].cuda() for k in ("x", "w", "bias"))
        if family.startswith("tc16"):
            c = lowp_conv1d(x, w, bias, precision=prec, in_slope=case.slope, dilation=case.dil, padding=case.padding,
                            transposed=bool(case.stride), stride=max(1, case.stride))
        else:
            c = _conv_ref(case, x, w, bias, torch.float64)
        _WANT64[key] = _epi_ref(case, c, inp)
    return _WANT64[key]


def _cpu32(case):
    """the same layer through torch's fp32 CPU conv, every epilogue step rounded to fp32"""
    if case.name not in _CPU32:
        inp = _inputs(case)
        _CPU32[case.name] = _epi_ref(case, _conv_ref(case, inp["x"], inp["w"], inp["bias"], torch.float32), inp)
    return _CPU32[case.name]


def _module(case, prec):
    from tts_b200.conv import FusedConv1d
    inp = _inputs(case)
    kw = dict(tensor_cores=False) if prec == "off" else dict(precision=prec)
    return FusedConv1d(inp["w"], inp["bias"], dilation=case.dil, padding=case.padding, transposed=bool(case.stride),
                       stride=max(1, case.stride), **kw)


def _launch_strided(case, conv):
    """One launch through b200tts_conv1d_forward_strided with NaN around the input and the output.  Returns
    (y, peak or None, dispatch names)."""
    from tts_b200 import _lib
    L = _lib.lib()
    inp, e = _inputs(case), EPI[case.epi]
    dev = torch.device("cuda:0")
    h = conv._handle(dev)
    b, cin, t = inp["x"].shape
    pitch, chans = -(-t // 4) * 4, cin + SPARE_CH
    xbuf = torch.full((b + 1, chans, pitch), NAN, device=dev)    # NaN pitch columns, spare channels, one spare batch row
    xbuf[:b, :cin, :t] = inp["x"].to(dev)
    tout = L.b200tts_conv1d_out_len(h, t)
    want_len = _want(case, case.family, "tf32x3").shape[-1]
    assert tout == want_len, f"b200tts_conv1d_out_len {tout} != torch's {want_len}"
    n = b * case.cout * tout
    ybuf = torch.full((GUARD + n + GUARD,), NAN, device=dev)
    y = ybuf[GUARD:GUARD + n].view(b, case.cout, tout)
    if inp["y_old"] is not None:
        y.copy_(inp["y_old"])
    res = None if inp["res"] is None else inp["res"].to(dev)
    peak = torch.zeros(1, dtype=torch.int32, device=dev) if e.get("tanh") else None
    with _lib.dispatch_log() as log:
        rc = L.b200tts_conv1d_forward_strided(h, _lib.ptr(xbuf), ctypes.c_longlong(chans * pitch), pitch, b, t,
                                              ctypes.c_float(case.slope), _lib.ptr(res), ctypes.c_float(e.get("scale", 1.0)),
                                              int(inp["y_old"] is not None), ctypes.c_float(e.get("post_div", 1.0)),
                                              int(bool(e.get("tanh"))), _lib.ptr(y), _lib.ptr(peak), _lib.stream_ptr(dev))
    _lib.check(rc, "conv1d_forward_strided")
    torch.cuda.synchronize()
    assert L.b200tts_debug_tc_error() == 0
    nan = torch.isnan(y)
    assert not nan.any(), f"{int(nan.sum())} output elements not written, first at {nan.nonzero()[0].tolist()}"
    assert torch.isnan(ybuf[:GUARD]).all() and torch.isnan(ybuf[GUARD + n:]).all(), "a guard element was overwritten"
    return y, peak, log.names


def _run(case, prec):
    """memoised strided launch of `case` at `prec` (the bit-exact comparisons reuse other precisions' results)"""
    key = (case.name, prec)
    if key not in _RUNS:
        conv = _module(case, prec)
        _RUNS[key] = (conv,) + _launch_strided(case, conv)
    return _RUNS[key]


def _record(prec, family, m):
    s = _STATS.setdefault((prec, family), dict(n=0, rel=0.0, col=0.0, row=0.0, max=0.0))
    s["n"] += 1
    for k in ("rel", "col", "row", "max"):
        s[k] = max(s[k], m[k])


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if _STATS:
        print("\nconv engine edges: measured maxima per (precision, family) -- rel RMS, worst column, worst row, max|err|/max")
        for (prec, fam), s in sorted(_STATS.items()):
            vs = (f"  err / fp32 CPU conv's: whole {s['vs_cpu'][0]:.2f} ({s['vs_cpu'][1]}), worst column "
                  f"{s['vs_cpu_col'][0]:.2f} ({s['vs_cpu_col'][1]})" if "vs_cpu" in s else "")
            print(f"  {prec:>6} {fam:<13} n={s['n']:3d}  rel {s['rel']:.2e}  col {s['col']:.2e}  row {s['row']:.2e}  "
                  f"max {s['max']:.2e}{vs}")


# ----------------------------------------------------------------------------- the sweep
@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_conv_engine_edge(case, prec):
    fam = expected_family(case, prec)
    conv, y, peak, names = _run(case, prec)
    assert names == [fam], f"dispatched {names}, expected [{fam!r}] ({case})"
    want = _want(case, fam, prec)

    fails, m = CC.failures(y, want, LAYER_REL_TOL)
    assert not fails, (case, fails)
    _record(prec if fam not in ("fma", "row1") else "fp32", fam, m)
    if fam in ("fma", "row1"):
        fails = CC.fp32_calibrated_failures(y, want, _cpu32(case))
        assert not fails, (case, fails)
        e = CC.fp32_errors(y, want, _cpu32(case))
        s = _STATS[("fp32", fam)]
        s["vs_cpu"] = max(s.get("vs_cpu", (0.0, "")), (e["got"] / max(e["cpu"], 1e-30), case.name))
        s["vs_cpu_col"] = max(s.get("vs_cpu_col", (0.0, "")), (e["got_col"] / max(e["cpu_col"], 1e-30), case.name))
    if peak is not None:   # the peak word is max|y|, bit for bit
        assert torch.equal(peak.view(torch.float32), y.abs().max().reshape(1)), (peak.view(torch.float32), y.abs().max())

    # bit-exact properties of the dispatch design
    if prec != "off" and fam == expected_family(case, "off"):
        assert torch.equal(y, _run(case, "off")[1]), "FMA fallback differs from the tensor_cores=False handle"
    if prec in ("f16x3", "bf16", "fp16") and case.cin % 16 and fam.startswith("tc3"):
        assert torch.equal(y, _run(case, "tf32x3")[1]), "Cin % 16 != 0 must run the 3xTF32 images"
    y2, peak2, names2 = _launch_strided(case, conv)
    assert names2 == names and torch.equal(y2, y), "a second launch differs from the first"

    # the contiguous call through FusedConv1d
    from tts_b200 import _lib
    inp, e = _inputs(case), EPI[case.epi]
    acc = None if inp["y_old"] is None else inp["y_old"].cuda()
    peak3 = torch.zeros(1, dtype=torch.int32, device="cuda") if e.get("tanh") else None
    with _lib.dispatch_log() as log:
        y3 = conv(inp["x"].cuda(), in_slope=case.slope, residual=None if inp["res"] is None else inp["res"].cuda(),
                  scale=e.get("scale", 1.0), accumulate_into=acc, post_div=e.get("post_div", 1.0),
                  tanh=bool(e.get("tanh")), peak=peak3)
    torch.cuda.synchronize()
    assert _lib.lib().b200tts_debug_tc_error() == 0
    fam3 = expected_family(case, prec, strided=False)
    assert log.names == [fam3], f"contiguous call dispatched {log.names}, expected [{fam3!r}]"
    if fam3 == fam:
        assert torch.equal(y3, y), "the contiguous call differs from the strided launch of the same family"
        if peak is not None:
            assert torch.equal(peak3, peak)
    else:   # unaligned rows: the FMA kernel, the same arithmetic as the tensor_cores=False handle
        assert torch.equal(y3, _run(case, "off")[1]), "the contiguous FMA call differs from the tensor_cores=False handle"
