"""The conv engine's internal prologue / epilogue options (``ConvIO``) against float64, one layer at a time.

test_conv_engine_edges_gpu.py covers what the public ``b200tts_conv1d_forward*`` calls expose.  The options below are
reachable only through the engines (and ``b200tts_debug_conv1d_create`` / ``_launch``): the WaveNet gate with per-row
``cond`` (interleaved by GEMM row, as WaveNet::init packs it), the res/skip split into y / y2, the masks, ReLU and
log-clamp, the coupling layers' channel flips, ragged rows, column windows and reflection padding.

Each case states the kernel family it runs on at tf32x3, derived from ``try_launch_tc`` / ``launch_conv`` (conv1d.cu):
  gate / split / ymask / mask_pre layers: tc3 with the general epilogue, never grouped (and FMA below Tq 128);
  ReLU or cond on 32 / 64 rows without ymask: tc3_grouped (the time-major kernel at f16x3, which logs as tc3_grouped);
  an input mask (xmask) or log-clamp: fma;  plain layers with cond: tc3's lean epilogue;
  tanh on one row, K 7, pad 3, Tout % 4 == 0: row1.
Every case runs at tf32x3, f16x3, bf16, fp16 and with tensor cores off (fma; row1 stays row1).  The input lives in a
NaN-filled pitched buffer (row pitch round_up(T, 4), spare channels and a spare batch row), every output inside NaN
guards, so an element not written or written out of place shows.

Bounds are the edge sweep's: LAYER_REL_TOL plus the per-slice checks of conv_check.py for every family,
lowp_reference for 16-bit operands, and for the FP32-FMA and row1 kernels the error of the same layer through torch's
fp32 CPU ops.  Masks hold zeros and ones only.  Bit-exact properties: a precision whose layer falls back to the FMA kernel
equals the tensor_cores=False handle; a relaunch equals the first launch; a ragged launch equals the dense one on every
column whose receptive field lies inside its row's extent; a windowed launch equals the dense one inside the window
(and, on the FMA and row1 kernels, writes nothing outside it).  The measured maxima are printed at the end (``-s``).
"""
import ctypes
import gc
import time
from dataclasses import dataclass

import pytest
import torch

import conv_check as CC
from lowp_reference import lowp_conv1d
from test_bench_scale_gpu import LAYER_REL_TOL

pytestmark = pytest.mark.gpu

PRECS = ["tf32x3", "f16x3", "bf16", "fp16", "off"]
SPARE_CH = 2
GUARD = 64
NAN = float("nan")
G, MP, MQ, AC, SP, A2 = CC.EPI_GATE, CC.EPI_MASK_PRE, CC.EPI_MASK_POST, CC.EPI_ACCUM, CC.EPI_SPLIT, CC.EPI_ACCUM2
RELU, TANH, LOGC = CC.ACT_RELU, CC.ACT_TANH, CC.ACT_LOGCLAMP


@dataclass(frozen=True)
class Case:
    name: str
    group: str           # option group of the report
    cin: int
    rows: int            # GEMM rows: Cout (a gate layer: 2H)
    k: int
    family: str          # at tf32x3: "tc3", "tc3_grouped", "fma" or "row1"
    dil: int = 1
    pad: int = -1        # -1: "same"
    b: int = 2
    t: int = 300
    slope: float = 1.0
    flags: int = 0
    act: int = 0
    act_param: float = 0.0
    cond: bool = False
    xmask: bool = False
    ymask: str = ""      # "tail": zeros at row ends; "holes": zeros inside the rows too
    split: int = 0
    res: bool = False
    scale: float = 1.0
    post_div: float = 1.0
    perm: str = ""       # "in" / "out": reversed input / output channel order (odd flow blocks)
    y_rows: int = 0      # > 0: y is rows [y_rows - Cout, y_rows) of a [B, y_rows, T] tensor (coupling post: z's x1)
    reflect: bool = False
    lens: tuple = ()     # ragged rows (b = len(lens))
    rate: int = 1        # rate_out = rate_in
    need: int = 0        # need_out; need_in = need + reach - pad, so every column below the extent is valid
    window: tuple = ()   # (q_lo, q_hi, in_lo, in_hi)
    fill: float = NAN    # windowed input outside [in_lo, in_hi)

    @property
    def padding(self):
        return self.dil * (self.k - 1) // 2 if self.pad < 0 else self.pad

    @property
    def batch(self):
        return len(self.lens) if self.lens else self.b

    @property
    def cout(self):      # rows of y (+ y2)
        return self.rows // 2 if self.flags & G else self.rows


C = Case
_g = torch.Generator().manual_seed(5)
LENS_TM_256 = tuple(int(v) for v in torch.randint(0, 301, (256,), generator=_g))
LENS_TM_300 = tuple(int(v) for v in torch.randint(0, 301, (300,), generator=_g))

CASES = [
    # ---- WaveNet gate (in_layer: 2H rows from H channels, K 5): partial row tiles (2H = 200, 400), a tile holding both
    #      halves (2H <= 128), Tq on either side of 128 / 256; per-row cond as the flow's WaveNet adds it
    C("gate_h16", "gate", 16, 32, 5, "tc3", t=301, flags=G, cond=True),
    C("gate_h64", "gate", 64, 128, 5, "tc3", t=301, flags=G, cond=True),
    C("gate_h96", "gate", 96, 192, 5, "tc3", t=301, flags=G, cond=True),
    C("gate_h192", "gate", 192, 384, 5, "tc3", t=301, flags=G, cond=True),
    C("gate_h200", "gate", 200, 400, 5, "tc3", t=301, flags=G, cond=True),
    C("gate_h100_nocond", "gate", 100, 200, 5, "tc3", t=301, flags=G),
    C("gate_h192_nocond", "gate", 192, 384, 5, "tc3", t=256, flags=G),
    C("gate_d2_tq127", "gate", 96, 192, 5, "fma", dil=2, t=127, flags=G, cond=True),
    C("gate_d2_tq128", "gate", 96, 192, 5, "tc3", dil=2, t=128, flags=G, cond=True),
    C("gate_d2_tq255", "gate", 96, 192, 5, "tc3", dil=2, t=255, flags=G, cond=True),
    C("gate_d2_tq256", "gate", 96, 192, 5, "tc3", dil=2, t=256, flags=G, cond=True),
    C("gate_d2_tq301", "gate", 96, 192, 5, "tc3", dil=2, t=301, flags=G, cond=True),
    C("gate_h32_d2", "gate", 32, 64, 5, "tc3", dil=2, t=257, flags=G, cond=True),   # 2H = 64: still never grouped
    # ---- WaveNet res/skip (1x1, 2H rows): the split at row 64 / 96 of the first tile, 64 of the second
    C("split_first_h64", "split", 64, 128, 1, "tc3", t=301, flags=SP, split=64, ymask="holes"),
    C("split_first_h96", "split", 96, 192, 1, "tc3", t=301, flags=SP, split=96, ymask="holes"),
    C("split_first_h192", "split", 192, 384, 1, "tc3", t=301, flags=SP, split=192, ymask="holes"),
    C("split_later_h64", "split", 64, 128, 1, "tc3", t=256, flags=SP | A2, split=64, ymask="holes"),
    C("split_later_h96", "split", 96, 192, 1, "tc3", t=301, flags=SP | A2, split=96, ymask="holes"),
    C("split_later_h192", "split", 192, 384, 1, "tc3", t=129, flags=SP | A2, split=192, ymask="holes"),
    C("split_later_h96_tq127", "split", 96, 192, 1, "fma", t=127, flags=SP | A2, split=96, ymask="holes"),
    C("split_last_h64", "split", 64, 64, 1, "tc3", t=301, flags=MQ | AC, ymask="holes"),
    C("split_last_h96", "split", 96, 96, 1, "tc3", t=301, flags=MQ | AC, ymask="holes"),
    C("split_last_h192", "split", 192, 192, 1, "tc3", t=301, flags=MQ | AC, ymask="holes"),
    # ---- coupling pre (h = pre(x0) * mask, reversed input channels) and post (x1 = (x1 -+ post(h) * mask) * mask,
    #      reversed output rows, y inside z: y_bs = 2 half T)
    C("coupling_pre", "coupling", 96, 192, 1, "tc3", t=301, flags=MQ, ymask="tail", perm="in"),
    C("coupling_pre_h32", "coupling", 16, 32, 1, "tc3", t=257, flags=MQ, ymask="holes", perm="in"),
    C("coupling_post_rev", "coupling", 192, 96, 1, "tc3", t=301, flags=MP | AC | MQ, ymask="holes", scale=-1.0,
      perm="out", y_rows=192),
    C("coupling_post_fwd", "coupling", 192, 96, 1, "tc3", t=301, flags=MP | AC | MQ, ymask="holes", scale=1.0,
      perm="out", y_rows=192),
    C("coupling_post_h64", "coupling", 192, 64, 1, "tc3", t=256, flags=MP | AC | MQ, ymask="tail", scale=-1.0,
      perm="out", y_rows=128),
    C("mask_pre_res", "coupling", 64, 96, 3, "tc3", t=301, flags=MP, ymask="holes", res=True, scale=0.5),
    C("mask_pre_res_div", "coupling", 64, 96, 3, "tc3", t=257, flags=MP | AC | MQ, ymask="holes", res=True,
      post_div=3.0),
    # ---- ReLU: FMA with an input mask (text encoder FFN), the general epilogue (ForwardTTS ffn1: 1536 rows), the
    #      grouped / time-major epilogues at 32 / 64 rows with cond
    C("relu_fma_xmask", "relu", 192, 192, 3, "fma", t=301, act=RELU, xmask=True, flags=MQ, ymask="tail"),
    C("relu_fma_xmask_k1", "relu", 80, 96, 1, "fma", t=130, act=RELU, xmask=True, slope=0.1),
    C("relu_ffn1", "relu", 384, 1536, 3, "tc3", t=203, act=RELU),
    C("relu_ffn1_mask", "relu", 384, 1536, 3, "tc3", t=203, act=RELU, flags=MQ, ymask="tail"),
    C("relu_g64_cond", "relu", 64, 64, 5, "tc3_grouped", t=301, act=RELU, cond=True),
    C("relu_g64_cond_res", "relu", 48, 64, 3, "tc3_grouped", t=481, act=RELU, cond=True, res=True, flags=AC),
    C("relu_g32_cond", "relu", 32, 32, 3, "tc3_grouped", t=257, act=RELU, cond=True, slope=0.1),
    C("relu_g32_cond_k7", "relu", 64, 32, 7, "tc3_grouped", t=300, act=RELU, cond=True),
    C("cond_g64", "relu", 64, 64, 3, "tc3_grouped", t=256, cond=True),
    C("relu_g64_ymask", "relu", 64, 64, 3, "tc3", t=301, act=RELU, flags=MQ, ymask="tail"),   # ymask: not grouped
    # ---- log-clamp (mel projection): values on both sides of act_param
    C("logclamp", "logclamp", 192, 80, 1, "fma", t=301, act=LOGC, act_param=0.05),
    C("logclamp_mask", "logclamp", 64, 80, 3, "fma", t=130, act=LOGC, act_param=0.05, flags=MQ, ymask="tail"),
    # ---- cond on the lean epilogue (HiFiGAN conv_pre with speaker conditioning)
    C("lean_cond_512", "lean_cond", 80, 512, 7, "tc3", t=512, cond=True),
    C("lean_cond_512_t301", "lean_cond", 80, 512, 7, "tc3", t=301, cond=True),
    C("lean_cond_res", "lean_cond", 64, 192, 3, "tc3", t=384, cond=True, res=True, flags=AC, slope=0.1),
    # ---- ragged rows: extents at tile boundaries +-1 (256 plain / time-major, 240 grouped, 128 time-major narrow),
    #      lens 0 and 1, rate / need other than 1 / 0
    C("ragged_lean", "ragged", 32, 96, 5, "tc3", t=300, res=True, lens=(257, 256, 255, 0, 1, 300, 129)),
    C("ragged_lean_rate", "ragged", 32, 96, 5, "tc3", t=300, res=True, lens=(128, 127, 0, 1, 150, 64), rate=2, need=3),
    C("ragged_gate", "ragged", 96, 192, 5, "tc3", t=300, flags=G, cond=True, lens=(257, 256, 255, 0, 1, 300)),
    C("ragged_split", "ragged", 96, 192, 1, "tc3", t=300, flags=SP | A2, split=96, ymask="tail",
      lens=(257, 256, 255, 0, 1, 300)),
    C("ragged_post", "ragged", 192, 96, 1, "tc3", t=300, flags=MP | AC | MQ, ymask="tail", scale=-1.0, perm="out",
      y_rows=192, lens=(257, 1, 0, 300)),
    C("ragged_g64", "ragged", 64, 64, 5, "tc3_grouped", t=481,
      lens=(241, 240, 239, 481, 0, 1, 257, 256, 129, 128, 480)),
    C("ragged_g32_rate", "ragged", 32, 32, 3, "tc3_grouped", dil=3, t=481, lens=(120, 119, 0, 1, 64, 63), rate=2,
      need=1),
    C("ragged_row1", "ragged", 32, 1, 7, "row1", t=1024, act=TANH, lens=(256, 255, 0, 1, 64, 63), rate=4),
    C("ragged_row1_need", "ragged", 16, 1, 7, "row1", t=1024, act=TANH, lens=(100, 33, 0, 1), rate=8, need=5),
    C("ragged_tm_b256", "ragged", 64, 64, 3, "tc3_grouped", t=300, lens=LENS_TM_256),
    C("ragged_tm_b300", "ragged", 64, 64, 3, "tc3_grouped", t=300, lens=LENS_TM_300),
    # ---- column windows (streaming): q_lo / q_hi off the tile grid, no data outside [in_lo, in_hi)
    C("window_lean", "window", 32, 96, 5, "tc3", dil=2, t=600, res=True, window=(37, 491, 33, 499)),
    C("window_gate", "window", 96, 192, 5, "tc3", t=600, flags=G, cond=True, window=(250, 263, 248, 265)),
    C("window_mask", "window", 96, 192, 1, "tc3", t=600, flags=MQ, ymask="holes", window=(129, 385, 129, 385)),
    C("window_g64", "window", 64, 64, 5, "tc3_grouped", t=600, window=(241, 479, 239, 481)),
    C("window_g32_big", "window", 32, 32, 3, "tc3_grouped", t=600, window=(130, 377, 128, 380), fill=1e6),
    C("window_plain_big", "window", 32, 96, 3, "tc3", t=600, window=(257, 511, 256, 512), fill=1e6),
    C("window_row1", "window", 32, 1, 7, "row1", t=1024, act=TANH, window=(101, 777, 98, 780)),
    # ---- reflection padding (MelGAN's pads) on the lean, grouped / time-major, row1 and FMA variants
    C("reflect_lean_k7", "reflect", 80, 256, 7, "tc3", t=256, reflect=True, slope=0.2),
    C("reflect_lean_k7_t257", "reflect", 80, 256, 7, "tc3", t=257, reflect=True, slope=0.2),
    C("reflect_g64_d9", "reflect", 64, 64, 3, "tc3_grouped", dil=9, t=256, reflect=True, slope=0.2),
    C("reflect_g64_d3_t481", "reflect", 64, 64, 3, "tc3_grouped", dil=3, t=481, reflect=True, slope=0.2),
    C("reflect_g32_d3", "reflect", 32, 32, 3, "tc3_grouped", dil=3, t=257, reflect=True, slope=0.2),
    C("reflect_row1", "reflect", 32, 1, 7, "row1", t=256, act=TANH, reflect=True, slope=0.2),
    C("reflect_row1_t4", "reflect", 32, 1, 7, "row1", t=4, act=TANH, reflect=True, slope=0.2),
    C("reflect_fma_d27", "reflect", 32, 32, 3, "fma", dil=27, t=127, reflect=True, slope=0.2),
    C("reflect_fma_limit", "reflect", 16, 24, 7, "fma", t=4, reflect=True, slope=0.2),   # pad 3 = Tin - 1
]
assert len({c.name for c in CASES}) == len(CASES)


def expected_family(case, prec):
    fam = case.family
    if fam in ("row1", "fma") or prec == "off":
        return fam if fam == "row1" else "fma"
    if prec in ("bf16", "fp16") and case.cin % 16 == 0:
        return fam.replace("tc3", "tc16")
    return fam


# ----------------------------------------------------------------------------- inputs and references
_INPUTS, _RUNS, _STATS = {}, {}, {}
_T0 = [None]


def _gate_row(r, h):         # logical row of a gate layer -> GEMM row (pack_conv's interleave)
    return 2 * r if r < h else 2 * (r - h) + 1


def _phys_rows(case):
    """GEMM row of every logical row (cond is indexed by it)"""
    if case.flags & G:
        return [_gate_row(r, case.rows // 2) for r in range(case.rows)]
    if case.perm == "out":
        return list(reversed(range(case.rows)))
    return list(range(case.rows))


def _tout(case):
    return case.t + 2 * case.padding - case.dil * (case.k - 1)


def _inputs(case):
    v = _INPUTS.get(case.name)
    if v is not None:
        return v
    g = torch.Generator().manual_seed(sum(map(ord, case.name)))
    B, T, To = case.batch, case.t, _tout(case)
    x = torch.randn(B, case.cin, T, generator=g)                       # logical channel order
    w = torch.randn(case.rows, case.cin, case.k, generator=g) / (case.cin * case.k) ** 0.5
    bias = torch.randn(case.rows, generator=g) * 0.1
    cond = torch.randn(B, case.rows, generator=g) * 0.5 if case.cond else None
    xmask = (torch.arange(T)[None, :] < torch.randint(T // 2, T + 1, (B, 1), generator=g)).float() if case.xmask else None
    ymask = None
    if case.ymask:
        ymask = (torch.arange(To)[None, :] < torch.randint(To // 2, To, (B, 1), generator=g)).float()
        ymask[:, 0] = 1
        if case.ymask == "holes":
            ymask[0, 3:9] = 0
            ymask[-1, To // 3: To // 3 + 5] = 0
    n_y = case.split if case.flags & SP else case.cout
    res = torch.randn(B, case.cout, To, generator=g) if case.res else None
    y_old = torch.randn(B, n_y, To, generator=g) if (case.flags & (AC | SP)) else None
    y2_old = torch.randn(B, case.rows - case.split, To, generator=g) if case.flags & A2 else None
    v = _INPUTS[case.name] = dict(x=x, w=w, bias=bias, cond=cond, xmask=xmask, ymask=ymask, res=res, y_old=y_old,
                                  y2_old=y2_old)
    return v


_REFS = {}


def _reference(case, family, prec, dtype=torch.float64, device="cuda"):
    """(y, y2) of the layer in logical row order: float64 (lowp_reference for 16-bit operands), or with dtype float32 on
    the CPU every step rounded to fp32"""
    key = (case.name, prec if family.startswith("tc16") else "", dtype, device)
    if key not in _REFS:
        _REFS[key] = _reference_uncached(case, family, prec, dtype, device)
    return _REFS[key]


def _reference_uncached(case, family, prec, dtype, device):
    inp = _inputs(case)
    dev = torch.device(device)
    t = {k: (None if v is None else v.to(dev)) for k, v in inp.items()}
    conv_fn = None
    if family.startswith("tc16"):
        def conv_fn(xm, slope, padding):
            return lowp_conv1d(xm, t["w"], t["bias"], precision=prec, in_slope=slope, dilation=case.dil, padding=padding)
    flags = case.flags
    return CC.engine_layer(t["x"], t["w"], t["bias"], dilation=case.dil, padding=case.padding, reflect=case.reflect,
                           xmask=t["xmask"], in_slope=case.slope, dtype=dtype, conv_fn=conv_fn, cond=t["cond"],
                           act=case.act, act_param=case.act_param, ymask=t["ymask"], flags=flags, residual=t["res"],
                           scale=case.scale, y_old=t["y_old"], post_div=case.post_div, split=case.split,
                           y2_old=t["y2_old"])


def _handle(case, prec):
    from tts_b200 import _lib
    inp = _inputs(case)
    cfg = _lib.Conv1dConfigC(case.cin, case.rows, case.k, case.dil, case.padding, 0, 1)
    w = inp["w"].contiguous()
    b = inp["bias"].contiguous()
    rev_in = torch.arange(case.cin - 1, -1, -1, dtype=torch.int32)
    rev_out = torch.arange(case.rows - 1, -1, -1, dtype=torch.int32)
    out = ctypes.c_void_p()
    tc = prec != "off"
    rc = _lib.lib().b200tts_debug_conv1d_create(
        ctypes.byref(cfg), _lib.ptr(w), _lib.ptr(b), int(tc), _lib.precision_id(prec if tc else "fp32"),
        int(case.reflect), case.rows // 2 if case.flags & G else 0,
        _lib.ptr(rev_in) if case.perm == "in" else None, _lib.ptr(rev_out) if case.perm == "out" else None,
        ctypes.byref(out))
    _lib.check(rc, "debug_conv1d_create")
    return out


class _Handle:
    def __init__(self, case, prec):
        from tts_b200 import _lib
        self.lib = _lib.lib()
        self.h = _handle(case, prec)

    def __del__(self):
        self.lib.b200tts_conv1d_destroy(self.h)


def _same(a, b):
    """bit for bit, NaN (a column a launch does not write) included"""
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _launch(case, handle, ragged=True, windowed=True):
    """One launch through b200tts_debug_conv1d_launch.  Returns (y, y2 or None, dispatch names, raw output buffers) with
    y / y2 in logical row order."""
    from tts_b200 import _lib
    L = _lib.lib()
    inp = _inputs(case)
    dev = torch.device("cuda:0")
    B, T, To = case.batch, case.t, _tout(case)
    assert L.b200tts_conv1d_out_len(handle.h, T) == To
    pitch, chans = -(-T // 4) * 4, case.cin + SPARE_CH
    xbuf = torch.full((B + 1, chans, pitch), NAN, device=dev)
    xs = inp["x"].flip(1) if case.perm == "in" else inp["x"]         # physical channel perm[c] holds logical c
    if windowed and case.window:
        q_lo, q_hi, in_lo, in_hi = case.window
        xbuf[:B, :case.cin, :T] = case.fill
        xbuf[:B, :case.cin, in_lo:in_hi] = xs[:, :, in_lo:in_hi].to(dev)
    else:
        xbuf[:B, :case.cin, :T] = xs.to(dev)
    io = _lib.DebugConvIOC()
    io.x, io.x_batch_stride, io.x_channel_stride, io.T = xbuf.data_ptr(), chans * pitch, pitch, T
    io.in_slope, io.scale, io.post_div = case.slope, case.scale, case.post_div
    io.act, io.act_param, io.flags, io.B, io.split = case.act, case.act_param, case.flags, B, case.split
    io.rate_out = io.rate_in = case.rate
    io.q_lo, io.q_hi, io.in_lo, io.in_hi = 0, 0x7fffffff, 0, 0x7fffffff
    keep = [xbuf]
    if inp["xmask"] is not None:
        xm = inp["xmask"].to(dev).contiguous()
        keep.append(xm)
        io.xmask, io.xmask_batch_stride = xm.data_ptr(), T
    if inp["cond"] is not None:
        cpitch = case.rows + 8
        cb = torch.full((B, cpitch), NAN, device=dev)
        cb[:, torch.tensor(_phys_rows(case))] = inp["cond"].to(dev)
        keep.append(cb)
        io.cond, io.cond_batch_stride = cb.data_ptr(), cpitch
    if inp["ymask"] is not None:
        ym = inp["ymask"].to(dev).contiguous()
        keep.append(ym)
        io.ymask, io.ymask_batch_stride = ym.data_ptr(), To
    # y: [B, y_rows, To] with this layer's rows last (coupling post: x1 of z), NaN everywhere else, guards around
    n_y = case.split if case.flags & SP else case.cout
    y_rows = case.y_rows or n_y
    n = B * y_rows * To
    ybuf = torch.full((GUARD + n + GUARD,), NAN, device=dev)
    yall = ybuf[GUARD:GUARD + n].view(B, y_rows, To)
    y = yall[:, y_rows - n_y:]
    phys_y = list(reversed(range(n_y))) if case.perm == "out" else list(range(n_y))
    if inp["y_old"] is not None:
        y[:, torch.tensor(phys_y)] = inp["y_old"].to(dev)
    io.y, io.y_batch_stride, io.y_channel_stride = y.data_ptr(), y_rows * To, To
    y2buf = None
    if case.flags & SP:
        n2 = B * (case.rows - case.split) * To
        y2buf = torch.full((GUARD + n2 + GUARD,), NAN, device=dev)
        y2 = y2buf[GUARD:GUARD + n2].view(B, case.rows - case.split, To)
        if inp["y2_old"] is not None:
            y2.copy_(inp["y2_old"])
        io.y2, io.y2_batch_stride, io.y2_channel_stride = y2.data_ptr(), (case.rows - case.split) * To, To
    if inp["res"] is not None:
        r = inp["res"].to(dev).contiguous()
        r = r.flip(1) if case.perm == "out" else r
        r = r.contiguous()
        keep.append(r)
        io.res, io.res_batch_stride, io.res_channel_stride = r.data_ptr(), case.cout * To, To
    if ragged and case.lens:
        lt = torch.tensor(case.lens, dtype=torch.int32, device=dev)
        keep.append(lt)
        io.lens, io.need_out, io.need_in = lt.data_ptr(), case.need, case.need + case.dil * (case.k - 1) - case.padding
    if windowed and case.window:
        io.q_lo, io.q_hi, io.in_lo, io.in_hi = case.window
    with _lib.dispatch_log() as log:
        rc = L.b200tts_debug_conv1d_launch(handle.h, ctypes.byref(io), _lib.stream_ptr(dev))
    _lib.check(rc, "debug_conv1d_launch")
    torch.cuda.synchronize()
    assert L.b200tts_debug_tc_error() == 0
    for buf in (ybuf, y2buf):
        if buf is not None:
            assert torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[-GUARD:]).all(), "a guard element was overwritten"
    if y_rows > n_y:
        assert torch.isnan(yall[:, :y_rows - n_y]).all(), "rows of y outside the layer's were written"
    y_log = y[:, torch.tensor(phys_y)] if case.perm == "out" else y
    y2_log = None if y2buf is None else y2buf[GUARD:-GUARD].view(B, case.rows - case.split, To)
    return y_log.clone(), None if y2_log is None else y2_log.clone(), log.names


def _run(case, prec, ragged=True, windowed=True):
    key = (case.name, prec, ragged, windowed)
    if key not in _RUNS:
        h = _Handle(case, prec)
        _RUNS[key] = (h,) + _launch(case, h, ragged, windowed)
    return _RUNS[key]


def _record(prec, fam, group, m):
    s = _STATS.setdefault((prec, fam, group), dict(n=0, rel=0.0, col=0.0, row=0.0, max=0.0))
    s["n"] += 1
    for k in ("rel", "col", "row", "max"):
        s[k] = max(s[k], m[k])


@pytest.fixture(scope="module", autouse=True)
def _report():
    _T0[0] = time.time()
    yield
    if _STATS:
        n = sum(s["n"] for s in _STATS.values())
        print(f"\nconv engine epilogues: {n} checked outputs in {time.time() - _T0[0]:.0f} s; measured maxima per "
              "(precision, family, option group) -- rel RMS, worst column, worst row, max|err|/max")
        for (prec, fam, grp), s in sorted(_STATS.items()):
            vs = f"  err / fp32 CPU's: {s['vs_cpu'][0]:.2f} ({s['vs_cpu'][1]})" if "vs_cpu" in s else ""
            print(f"  {prec:>6} {fam:<13} {grp:<10} n={s['n']:3d}  rel {s['rel']:.2e}  col {s['col']:.2e}  "
                  f"row {s['row']:.2e}  max {s['max']:.2e}{vs}")
    # free the cached handles and device tensors here, not at some later garbage collection inside another module's
    # test (test_device_buffers_gpu.py counts the library's live device buffers)
    _RUNS.clear()
    _REFS.clear()
    gc.collect()


def _valid(case, out):
    """[B, T] bool: the columns this launch promises (ragged: below the row's extent; window: inside it)"""
    B, To = out.shape[0], out.shape[-1]
    v = torch.ones(B, To, dtype=torch.bool)
    if case.lens:
        v &= CC.columns_below(CC.ragged_extent(torch.tensor(case.lens), case.rate, case.need, To), To)
    if case.window:
        q = torch.arange(To)[None, :]
        v &= (q >= case.window[0]) & (q < case.window[1])
    return v.to(out.device)


def _check(case, fam, prec, got, want, cpu32, what):
    valid = _valid(case, got)[:, None, :]
    g = torch.where(valid, got.to(torch.float64), want)
    nan = torch.isnan(g)
    assert not nan.any(), f"{what}: {int(nan.sum())} promised elements not written, first at {nan.nonzero()[0].tolist()}"
    fails, m = CC.failures(g, want, LAYER_REL_TOL)
    assert not fails, (case.name, what, fails)
    fp32 = fam in ("fma", "row1")
    _record("fp32" if fp32 else prec, fam, case.group, m)
    if fp32:
        c32 = torch.where(valid.cpu(), cpu32, want.cpu().to(torch.float32))
        fails = CC.fp32_calibrated_failures(g, want, c32)
        assert not fails, (case.name, what, fails)
        e = CC.fp32_errors(g, want, c32)
        s = _STATS[("fp32", fam, case.group)]
        s["vs_cpu"] = max(s.get("vs_cpu", (0.0, "")), (e["got"] / max(e["cpu"], 1e-30), case.name))


# ----------------------------------------------------------------------------- the sweep
@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_conv_engine_epilogue(case, prec):
    fam = expected_family(case, prec)
    _, y, y2, names = _run(case, prec)
    assert names == [fam], f"dispatched {names}, expected [{fam!r}] ({case.name})"
    want, want2 = _reference(case, fam, prec)
    c32, c32_2 = _reference(case, fam, prec, torch.float32, "cpu") if fam in ("fma", "row1") else (None, None)
    _check(case, fam, prec, y, want, c32, "y")
    if want2 is not None:
        _check(case, fam, prec, y2, want2, c32_2, "y2")

    # bit-exact properties
    if prec != "off" and fam == expected_family(case, "off"):
        assert _same(y, _run(case, "off")[1]), "FMA fallback differs from the tensor_cores=False handle"
    h = _run(case, prec)[0]
    y_b, y2_b, names_b = _launch(case, h)
    assert names_b == names and _same(y_b, y) and (y2 is None or _same(y2_b, y2)), \
        "a second launch differs from the first"
    if case.lens or case.window:
        _, yd, yd2, names_d = _run(case, prec, ragged=False, windowed=False)
        assert names_d == names
        valid = _valid(case, y)[:, None, :]
        for got, dense in ((y, yd), (y2, yd2)):
            if got is None:
                continue
            assert _same(torch.where(valid, got, 0.0), torch.where(valid, dense, 0.0)), \
                "promised columns differ from the dense launch"
            if case.window and fam in ("fma", "row1"):
                assert torch.isnan(got[~valid.expand_as(got)]).all(), "a column outside the window was written"


# ----------------------------------------------------------------------------- combinations launch_conv rejects
@pytest.mark.parametrize("prec", ["tf32x3", "off"])
@pytest.mark.parametrize("what", ["ymask_without_flag", "ymask_with_gate", "gate_with_mask_flag", "gate_with_scale"])
def test_launch_conv_rejects_ignored_options(what, prec):
    """ymask without MASK_PRE / MASK_POST / SPLIT was applied by the FMA plain epilogue and ignored by the tensor-core
    general one; the gate epilogue ignored ymask, every other flag, scale and post_div.  launch_conv rejects them."""
    from dataclasses import replace
    from tts_b200 import _lib
    base = C(f"reject_{what}", "reject", 64, 128, 3, "tc3", t=256, flags=G if what != "ymask_without_flag" else 0, ymask="tail")
    case = {"ymask_without_flag": base, "ymask_with_gate": base,
            "gate_with_mask_flag": replace(base, flags=G | MQ),
            "gate_with_scale": replace(base, ymask="", scale=0.5)}[what]
    h = _Handle(case, prec)
    with pytest.raises(RuntimeError, match="status 1"):
        _launch(case, h)
    assert _lib.lib().b200tts_debug_tc_error() == 0
