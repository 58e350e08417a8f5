"""Checker for one layer of the conv engine against a float64 reference (``test_conv_engine_edges_gpu.py``).

A whole-tensor relative RMS cannot see one wrong output column or one row that lost its bias: at a few thousand
elements such an error is diluted below any sensible tolerance.  So the checker also bounds the error of every
(batch, output column) slice over all rows and of every (batch, row) slice over all columns, plus the largest single
error.  All of them are relative to the whole tensor's RMS (or max) of the reference, so a slice whose reference is
close to zero does not blow up.  ``test_conv_checker_cpu.py`` shows on CPU tensors that these bounds reject a dropped
tap x channel product at either end of a row, a lost bias in a partial row tile, a shifted last column and a 1e-3
perturbation of one column, and that they accept a 1e-6 random perturbation.

For the FP32-FMA kernel there is no measured absolute bound; its error is instead compared with the error torch's own
fp32 CPU conv makes on the same inputs (``fp32_calibrated_failures``).

Test infrastructure only, like ``lowp_reference.py``; it works on whatever device its inputs live on.
"""
import torch
import torch.nn.functional as F

SLICE_FACTOR = 2.0      # per-slice bound = SLICE_FACTOR x the whole-tensor bound (a starting value, not a measured one)
MAX_ABS_TOL = 2e-4      # max |err| <= MAX_ABS_TOL * max |want|, as the other layer tests
FMA_FACTOR = 8.0        # FP32-FMA kernel: within FMA_FACTOR x the error of torch's fp32 CPU conv ...
FMA_FLOOR = 2.0 ** -23  # ... plus FMA_FLOOR * max |want| (one fp32 ulp, for outputs the CPU conv happens to get exact)


def conv(x, w, bias=None, *, dilation=1, padding=0, transposed=False, stride=1, in_slope=1.0, dtype=torch.float64):
    """conv1d (w [Cout, Cin, K]) or conv_transpose1d (w [Cin, Cout, K]) of leaky_relu(x, in_slope), bias included,
    computed in ``dtype``."""
    xs = F.leaky_relu(x.to(dtype), in_slope)
    wd = w.to(dtype)
    b = None if bias is None else bias.to(dtype)
    if transposed:
        return F.conv_transpose1d(xs, wd, b, stride=stride, padding=padding)
    return F.conv1d(xs, wd, b, dilation=dilation, padding=padding)


def epilogue(c, *, residual=None, scale=1.0, y_old=None, post_div=1.0, tanh=False):
    """The engine's epilogue on a conv result ``c`` (bias included), in c's dtype and in the documented order
    ``((c + residual) * scale [+ y_old]) / post_div``, or ``tanh(c)``."""
    if tanh:
        return torch.tanh(c)
    if residual is not None:
        c = c + residual.to(c.dtype)
    if scale != 1.0:
        c = c * scale
    if y_old is not None:
        c = c + y_old.to(c.dtype)
    if post_div != 1.0:
        c = c / post_div
    return c


ACT_NONE, ACT_RELU, ACT_TANH, ACT_LOGCLAMP = 0, 1, 2, 3
EPI_GATE, EPI_MASK_PRE, EPI_MASK_POST, EPI_ACCUM, EPI_SPLIT, EPI_ACCUM2 = 1, 2, 4, 8, 16, 32


def engine_prologue(x, xmask=None, in_slope=1.0, dtype=torch.float64):
    """The engine's conv prologue in ``dtype``: x *= xmask[b, t] (xmask [B, T]), then leaky ReLU."""
    x = x.to(dtype)
    if xmask is not None:
        x = x * xmask.to(dtype)[:, None, :]
    return F.leaky_relu(x, in_slope)


def engine_epilogue(c, *, cond=None, act=ACT_NONE, act_param=0.0, ymask=None, flags=0, residual=None, scale=1.0,
                    y_old=None, post_div=1.0, split=0, y2_old=None):
    """The engine's epilogue (common.cuh, launch_conv) on a conv result ``c`` [B, R, T] with its bias, in c's dtype and
    in the documented order; returns (y, y2).  Rows are logical rows (a gate layer's first R/2 rows are the tanh half);
    cond [B, R] in the same order; ymask [B, T]; y_old / y2_old are the destinations' previous contents.
      v = c + cond;  gate: tanh(v[:H]) * sigmoid(v[H:]) (nothing else applies)  |  act
      mask_pre; + residual; * scale; + y_old (ACCUM); / post_div; mask_post
      split: rows < split -> y with ACCUM and MASK_POST forced on, rows >= split -> y2 (+ y2_old with ACCUM2, no mask)"""
    dt = c.dtype
    v = c if cond is None else c + cond.to(dt)[:, :, None]
    if flags & EPI_GATE:
        h = v.shape[1] // 2
        return torch.tanh(v[:, :h]) * torch.sigmoid(v[:, h:]), None
    if act == ACT_RELU:
        v = torch.relu(v)
    elif act == ACT_TANH:
        v = torch.tanh(v)
    elif act == ACT_LOGCLAMP:
        v = torch.log(torch.clamp_min(v, act_param))
    m = None if ymask is None else ymask.to(dt)[:, None, :]
    rows = v.shape[1]
    n_y = split if flags & EPI_SPLIT else rows
    accum = torch.zeros(rows, dtype=torch.bool)
    mpost = torch.zeros(rows, dtype=torch.bool)
    accum[:n_y], mpost[:n_y] = bool(flags & EPI_ACCUM) or n_y < rows, bool(flags & EPI_MASK_POST) or n_y < rows
    accum[n_y:] = bool(flags & EPI_ACCUM2)
    if flags & EPI_MASK_PRE:
        v = v * m
    if residual is not None:
        v = v + residual.to(dt)
    v = v * scale
    old = torch.zeros_like(v)
    if y_old is not None:
        old[:, :n_y] = y_old.to(dt)[:, :n_y]
    if y2_old is not None and n_y < rows:
        old[:, n_y:] = y2_old.to(dt)
    v = torch.where(accum[None, :, None].to(v.device), v + old, v)
    v = v / post_div
    if m is not None:
        v = torch.where(mpost[None, :, None].to(v.device), v * m, v)
    return v[:, :n_y], (v[:, n_y:] if n_y < rows else None)


def engine_layer(x, w, bias, *, dilation=1, padding=0, reflect=False, xmask=None, in_slope=1.0, dtype=torch.float64,
                 conv_fn=None, **epi):
    """One engine layer: engine_prologue, conv1d (w [R, Cin, K], logical rows; reflect: ReflectionPad1d(padding) and no
    zero padding) + bias, engine_epilogue(**epi); returns (y, y2).  ``conv_fn(x, in_slope, padding)`` replaces the
    leaky ReLU and the conv (lowp_reference for 16-bit operands); it gets x after the input mask and any reflection."""
    if conv_fn is not None:
        xm = x if xmask is None else x * xmask.to(x.dtype)[:, None, :]
    else:
        xm = engine_prologue(x, xmask, in_slope, dtype)
    if reflect and padding:
        xm = F.pad(xm, (padding, padding), mode="reflect")
        padding = 0
    if conv_fn is None:
        c = F.conv1d(xm, w.to(dtype), None if bias is None else bias.to(dtype), dilation=dilation, padding=padding)
    else:
        c = conv_fn(xm, in_slope, padding)
    return engine_epilogue(c, **epi)


def ragged_extent(lens, rate, need, limit):
    """ConvIO's ragged extent per row: min(limit, max(0, lens[b] * rate + need)), as a CPU int64 tensor"""
    return (lens.to(torch.int64).cpu() * rate + need).clamp(0, limit)


def columns_below(ext, T):
    """[B, T] bool: column t of row b is below ext[b]"""
    return torch.arange(T)[None, :] < ext[:, None]


def measure(got, want):
    """Relative errors of ``got`` [B, R, T] against ``want``: whole tensor, worst (batch, column), worst (batch, row)
    (RMS over the other axis, relative to the whole tensor's RMS) and worst element (relative to max |want|)."""
    err = got.to(torch.float64) - want.to(torch.float64)
    want = want.to(torch.float64)
    ref = float(want.pow(2).mean().sqrt().clamp_min(1e-30))
    col = err.pow(2).mean(dim=1).sqrt() / ref     # [B, T]
    row = err.pow(2).mean(dim=2).sqrt() / ref     # [B, R]
    ci, ri = int(col.argmax()), int(row.argmax())
    return {
        "rel": float(err.pow(2).mean().sqrt()) / ref,
        "col": float(col.max()), "col_at": divmod(ci, col.shape[1]),
        "row": float(row.max()), "row_at": divmod(ri, row.shape[1]),
        "max": float(err.abs().max()) / max(float(want.abs().max()), 1e-30),
    }


def failures(got, want, rel_tol, slice_factor=SLICE_FACTOR, max_tol=MAX_ABS_TOL):
    """(failed criteria, measured errors): whole-tensor relative RMS <= rel_tol, every (batch, column) and (batch, row)
    slice <= slice_factor * rel_tol, max |err| <= max_tol * max |want|."""
    if got.shape != want.shape:
        return [f"shape {tuple(got.shape)} != {tuple(want.shape)}"], {}
    m = measure(got, want)
    out = []
    if not m["rel"] <= rel_tol:
        out.append(f"whole-tensor rel RMS {m['rel']:.3e} > {rel_tol:.1e}")
    if not m["col"] <= slice_factor * rel_tol:
        out.append(f"per-column rel RMS {m['col']:.3e} at (batch, column) {m['col_at']} > {slice_factor * rel_tol:.1e}")
    if not m["row"] <= slice_factor * rel_tol:
        out.append(f"per-row rel RMS {m['row']:.3e} at (batch, row) {m['row_at']} > {slice_factor * rel_tol:.1e}")
    if not m["max"] <= max_tol:
        out.append(f"max abs err {m['max']:.3e} x max|want| > {max_tol:.1e}")
    return out, m


def fp32_errors(got, want, cpu32):
    """RMS error of ``got`` and of ``cpu32`` against the float64 ``want``, over the whole tensor and in the worst
    (batch, column) slice (RMS over rows), and where got's worst column is."""
    want = want.to(torch.float64)
    eg = got.to(torch.float64) - want
    ec = cpu32.to(torch.float64).to(want.device) - want
    cg, cc = eg.pow(2).mean(dim=1).sqrt(), ec.pow(2).mean(dim=1).sqrt()
    return {"got": float(eg.pow(2).mean().sqrt()), "cpu": float(ec.pow(2).mean().sqrt()),
            "got_col": float(cg.max()), "cpu_col": float(cc.max()), "col_at": divmod(int(cg.argmax()), cg.shape[1])}


def fp32_calibrated_failures(got, want, cpu32, factor=FMA_FACTOR, floor=FMA_FLOOR):
    """Failed criteria of an FP32 result: its error against the float64 ``want`` must stay within ``factor`` x the
    error of ``cpu32`` (the same layer through torch's fp32 CPU conv) plus ``floor`` * max |want|, over the whole
    tensor and in its worst (batch, column) slice."""
    fl = floor * float(want.abs().max())
    e = fp32_errors(got, want, cpu32)
    out = []
    if not e["got"] <= factor * e["cpu"] + fl:
        out.append(f"whole-tensor RMS err {e['got']:.3e} > {factor} x fp32 CPU conv's {e['cpu']:.3e} + {fl:.1e}")
    if not e["got_col"] <= factor * e["cpu_col"] + fl:
        out.append(f"worst column RMS err {e['got_col']:.3e} at (batch, column) {e['col_at']} > {factor} x fp32 CPU "
                   f"conv's {e['cpu_col']:.3e} + {fl:.1e}")
    return out
