"""Reference for one conv layer with 16-bit tensor-core operands (``precision="bf16"`` / ``"fp16"``).

What the kernel computes, up to fp32 accumulation order: the leaky ReLU is applied in fp32, its result is rounded to
the 16-bit type (round to nearest even), the weight (weight norm already folded, in fp32) is rounded the same way, and
the products are summed -- here in float64.  Bias and every epilogue term stay at full precision.  Test infrastructure
only, like oracle/vits_oracle.py; it works on whatever device its inputs live on.
"""
import torch
import torch.nn.functional as F

DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}


def round_to(x, precision):
    """fp32 values rounded to the 16-bit type (nearest even), returned as float64."""
    return x.to(torch.float32).to(DTYPES[precision]).to(torch.float64)


def lowp_conv1d(x, w, bias=None, *, precision, in_slope=1.0, dilation=1, padding=0, transposed=False, stride=1):
    """conv1d (w [Cout, Cin, K]) or conv_transpose1d (w [Cin, Cout, K]) of leaky_relu(x, in_slope), float64 result."""
    xs = x.to(torch.float32)
    xs = torch.maximum(xs, xs * in_slope)           # leaky ReLU as the kernel forms it (0 <= in_slope <= 1)
    xr, wr = round_to(xs, precision), round_to(w, precision)
    b = None if bias is None else bias.to(torch.float64)
    if transposed:
        return F.conv_transpose1d(xr, wr, b, stride=stride, padding=padding)
    return F.conv1d(xr, wr, b, dilation=dilation, padding=padding)
