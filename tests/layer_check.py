"""fp64 reference convs and the bf16-split error emulation shared by the per-layer tests
(test_backbone_layers.py, test_stage_layers.py).

The tensor-core kernels keep every fp32 operand as a bf16 pair (hi, lo) and accumulate the three
products x_hi w_hi + x_lo w_hi + x_hi w_lo in fp32.  For a layer and its actual input, ``e3`` is
the error that split commits in exact accumulation, ``e2`` the smaller error of its two 2-term
variants (one lo term dropped).  A layer passes when its error is below
``layer_bound(e3, K) = max(K_E3 * e3, FLOOR_C * sqrt(K) * 2^-24)``, and that bound must stay at
least ``SEPARATION`` times below ``e2``, so no bound can admit a lost term.

Geometry of a conv, the keyword arguments ``g`` of the functions below: ``stride`` and ``pad``
(an int or one value per spatial axis), ``transposed`` (k3, stride 2, pad 1, output pad 1, as
every transposed conv of the project), and ``region``: per spatial axis ``(lo, hi)`` output
indices or None for the whole axis.  A 4-D input is a 2-D conv, a 5-D input a 3-D conv; all
kernels are 3 wide.
"""
import math

import torch
import torch.nn.functional as F

from oracle import dfm_oracle as O

# 3-term error -> bound, and the margin the bound must keep below a lost term.  K_E3 was chosen
# from the measured H100 errors (DESIGN.md section 1, per-layer tables).
K_E3 = 6.0
SEPARATION = 3.0
U32 = 2.0 ** -24       # fp32 unit roundoff
FLOOR_C = 4.0          # fp32 accumulation floor: FLOOR_C * sqrt(K) * u


def acc_floor(k, floor_c=FLOOR_C):
    return floor_c * math.sqrt(k) * U32


def layer_bound(e3, k, floor_c=FLOOR_C):
    return max(K_E3 * e3, acc_floor(k, floor_c))


def _per_axis(v, nd):
    return tuple(v) if isinstance(v, (tuple, list)) else (v,) * nd


def window(x, stride=1, pad=1, region=None):
    """The zero-padded input window [1, Cin, *S'] that the outputs `region` of an unpadded
    k3 conv with `stride` read (only that window is copied: regions of large volumes stay
    cheap)."""
    nd = x.dim() - 2
    st, pd = _per_axis(stride, nd), _per_axis(pad, nd)
    region = tuple(region) if region is not None else (None,) * nd
    sl, widths = [slice(None), slice(None)], []
    for a in range(nd):
        n = x.shape[2 + a]
        lo, hi = region[a] or (0, (n + 2 * pd[a] - 3) // st[a] + 1)
        i0, i1 = st[a] * lo - pd[a], st[a] * (hi - 1) - pd[a] + 3
        sl.append(slice(max(i0, 0), min(i1, n)))
        widths.append((max(0, -i0), max(0, i1 - n)))
    return F.pad(x[tuple(sl)], [v for a in reversed(range(nd)) for v in widths[a]])


def _conv_t(x, w, region):
    nd = x.dim() - 2
    conv = F.conv_transpose3d if nd == 3 else F.conv_transpose2d
    region = tuple(region) if region is not None else (None,) * nd
    assert all(r is None for r in region[1:])
    if region[0] is None:
        return conv(x, w, None, 2, 1, 1)
    z0, z1 = region[0]
    assert z0 % 2 == 0
    i0, i1 = z0 // 2, min(z1 // 2 + 1, x.shape[2])
    return conv(x[:, :, i0:i1], w, None, 2, 1, 1)[:, :, :z1 - z0]


def conv_planes(x, w, stride=1, pad=1, transposed=False, region=None):
    """The outputs `region` of a k3 conv (conv_transpose k3 s2 p1 op1 if transposed) of the
    whole input x [1, Cin, *S], computed from the input window those outputs read (halo
    included, zero padding outside x).  For transposed convs only the first spatial axis may be
    restricted, to an even lo."""
    if transposed:
        return _conv_t(x, w, region)
    return tap_conv(window(x, stride, pad, region), w, _per_axis(stride, x.dim() - 2))


def tap_conv(x, w, stride):
    """Unpadded k3 conv of x [1, Cin, *S] as a sum over the taps of channels-last matrix
    products (fp64 GEMMs: far faster than a direct fp64 conv on large volumes)."""
    nd = x.dim() - 2
    xl = x[0].movedim(0, -1)                      # [*S, Cin]
    so = [(n - 3) // s + 1 for n, s in zip(x.shape[2:], stride)]
    y = x.new_zeros(so + [w.shape[0]])
    for tap in range(3 ** nd):
        k = [(tap // 3 ** (nd - 1 - a)) % 3 for a in range(nd)]
        sl = tuple(slice(k[a], k[a] + stride[a] * (so[a] - 1) + 1, stride[a]) for a in range(nd))
        y += xl[sl].reshape(-1, xl.shape[-1]).matmul(w[(Ellipsis,) + tuple(k)].t()) \
            .view(y.shape)
    return y.movedim(-1, 0)[None]


def k_of(cin, transposed=False, nd=3):
    """Products per output of a k3 conv (a transposed stride-2 conv reaches 2^nd taps)."""
    return cin * (2 ** nd if transposed else 3 ** nd)


def split16(x):
    """The bf16 (hi, lo) pair the kernels keep of an fp32 operand."""
    x = x.float()
    hi = O.bf16_round(x)
    return hi.double(), O.bf16_round(x - hi).double()


def emulated_outputs(x, w, stride=1, pad=1, transposed=False, region=None):
    """The 3-term split x_hi w_hi + x_lo w_hi + x_hi w_lo and its two 2-term variants (x_lo
    term dropped, w_lo term dropped), in exact (fp64) accumulation."""
    if transposed:
        def conv(a, b):
            return _conv_t(a, b, region)
    else:
        x = window(x, stride, pad, region)

        def conv(a, b):
            return tap_conv(a, b, _per_axis(stride, x.dim() - 2))
    xh, xl = split16(x)
    wh, wl = split16(w)
    a = conv(xh, wh)
    b = conv(xl, wh)
    c = conv(xh, wl)
    return a + b + c, a + c, a + b


def norm_errors(ys, ref):
    """(e3, e2): normalised max-norm error of the 3-term split and of the better 2-term variant
    (ys = emulated_outputs) against ref."""
    y3, y2x, y2w = ys
    s = float(ref.abs().max())
    e3 = float((y3 - ref).abs().max()) / s
    e2 = min(float((y2x - ref).abs().max()), float((y2w - ref).abs().max())) / s
    return e3, e2


def emulate(x, w, ref, **g):
    """(e3, e2) of the conv of x with w (geometry g) against ref = its exact outputs."""
    return norm_errors(emulated_outputs(x, w, **g), ref)


def product_scale(x, w, **g):
    """sum |x| |w| over each output's products: the scale of that output's rounding error,
    which stays meaningful where the output itself is small (z ends, zero-padded halo)."""
    return conv_planes(x.abs(), w.abs(), **g)


def elementwise_errors(got, ref, y3, y2x, y2w, scale, k, floor_c=FLOOR_C):
    """Element-wise form of the layer bound: the worst |a - ref| / scale over the elements
    given, for the GPU (a = got), the 3-term split and the better 2-term variant, and the bound
    max(K_E3 * e3, floor) that the GPU ratio must meet.  Returns (gpu, e3, e2, bound)."""
    s = scale.clamp_min(1e-12 * float(scale.max()))

    def worst(a):
        return float(((a - ref).abs() / s).max())
    e3 = worst(y3)
    return worst(got), e3, min(worst(y2x), worst(y2w)), layer_bound(e3, k, floor_c)
