"""Float64 op-list interpreter and per-element checker for one forward pass of a ``DeviceModel``.

Every op of ``cm.records`` is recomputed in float64 from the buffers the device itself produced (fetched by buffer id
through ``sb_model_forward``) and compared element by element with the device's output, against a bound derived from
how the kernel rounds (``elem_bound``), not from the map's maximum.  So each op is checked in isolation and no error can
hide behind the layers after it.

Operands are the ones each kernel actually uses (``sb_model_profile_ops`` kind 1 = tensor core, 2 = CUDA core):
  * tensor-core convs (wgmma, ``mma.sync`` heads, the Toeplitz / space-to-depth views, conv1 of ``k_conv01``):
    fp16(w) from the fp32 blob; ``k_conv_direct`` / ``k_conv_first`` / ``k_tconv_direct``: the fp32 blob;
  * a first conv fused with PREPROCESS reads the frame: ``k_conv_first`` the fp32 value, the views and ``k_conv01``
    fp16(value).  PREPROCESS itself is an exact sequence of fp32 operations (with the truncating u8 gray round trip), so
    its reference is that sequence replayed in numpy float32 (``preprocess32``), not a float64 recompute.
Precision 2 works on the physical ``[lo | hi | hi]`` layout: records carry physical input channels, the blob holds the
expanded ``[Wh | Wl | Wh]`` rows, a producer's slice is decoded as lo + hi (planes ``out_C`` apart) and its layout
invariants are asserted exactly.
Precision 1 (the fp32 CUDA-core path) keeps every buffer in fp32 and runs every conv on ``k_conv_direct`` /
``k_tconv_direct`` with the fp32 blob: no first-conv fusion, no tensor-core plan, so no fused pool or ADD either.  Its
elementwise ops have their own bounds (``elementwise_bound``).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from sleap_b200.nn import oplist as ol

ACC_ULP = 2.0 ** -23       # one fp32 accumulator ulp, relative to the accumulator
EPI_ULP = 2.0 ** -22       # four fp32 roundings (residual, bias, BN multiply, BN add) of the epilogue
F16_MIN_NORMAL = 2.0 ** -14


def f16(x):
    return np.asarray(x, np.float64).astype(np.float16).astype(np.float64)


def ulp16(y):
    """Spacing of fp16 numbers at |y| (2^-24 in the subnormal range)."""
    _, e = np.frexp(np.maximum(np.abs(y), F16_MIN_NORMAL))
    return np.ldexp(1.0, e - 11)


def out_rounding(ref, e_pre, out):
    """Error of the final store of a value known to within e_pre: fp16 rounds to nearest (1/2 ulp); the split store keeps
    hi + fp16(v - hi), 2^-22 relative (plus half the smallest lo subnormal); fp32 1/2 ulp; 'exact' none."""
    mag = np.abs(ref) + e_pre
    if out == "f16":
        return 0.5 * ulp16(mag)
    if out == "split":
        return 2.0 ** -22 * mag + 2.0 ** -25
    if out == "f32":
        return 2.0 ** -24 * mag
    return np.zeros_like(mag)


def elem_bound(A, mag, n_steps, prop=0.0, bn_scale=None, bn_mag=None):
    """Per-element bound on |device value before its final store - float64 value|, from the kernel's arithmetic.

    A       = sum |w| |x| over the element's products (the same conv on absolute values);
    mag     = |s| + |bias| + |residual| (s = sum w x);
    n_steps = accumulation steps that feed the element: K = 16 steps for wgmma / mma.sync, taps x C_in fma for the CUDA
              cores.  DESIGN 5.7: the tensor-core fp32 accumulator truncates, each step losing at most one ulp of the
              accumulator, and |accumulator| <= A; an fma rounds, half an ulp.  So E_acc = n_steps 2^-23 A;
    prop    = sum |w| E_in: the error of an input that is not visible (inside a fused chain), E_in being that stage's own
              bound including its fp16 rounding (2^-11 relative);
    epilogue: up to four fp32 roundings of magnitude <= mag; ReLU is 1-Lipschitz; a BN affine after it scales the
              error by |scale| and adds two roundings of |v scale| + |shift| (bn_mag).
    The final store (out_rounding) comes on top."""
    e = n_steps * ACC_ULP * A + prop + EPI_ULP * mag
    if bn_scale is not None:
        e = np.abs(bn_scale) * e + 2.0 * 2.0 ** -24 * bn_mag
    return e


def elementwise_bound(kind, ref, x=None):
    """(e_pre, store kind) of an elementwise op of the fp32 path (k_maxpool2 / k_maxpool3s2 / k_upsample2 / k_add with
    T = float, sb_kernels_direct.cuh) whose float64 reference from the fp32 device inputs is ``ref``.  u = 2^-24, one
    fp32 rounding.
      * pool, pool3s2, nearest: the output is one of the inputs (fmaxf, a copy): exact, no store rounding;
      * add: v = a + b, one rounding of |a + b| (the 'f32' store term); a ReLU after it keeps the sign, so is exact;
      * bilinear: per axis lerp t = l + (r - l) w with w in {1/4, 3/4} (0 where the edge clamp makes l = r).  With M the
        largest |corner|: r - l rounds (<= u 2M), (r - l) w rounds (<= u 3/4 2M; exact for w = 1/4), the add rounds
        (<= u M), so each of tp, bt is within 2u M + 3/4 2u M + u M < 4u M; the outer lerp carries that (weights 1 - w, w)
        and adds 3/4 2u M + 3/4 2u M + u M = 4u M.  So e_pre = 8u M = 2^-21 M, which already holds the final add's
        rounding; the 'f32' store term on top absorbs the second-order terms.  nvcc may contract (r - l) w + l into one
        FMA, which drops a rounding.
    ``x`` is the bilinear upsample's input map (M is taken over its 3 x 3 neighbourhood, which holds all four corners)."""
    if kind in ("pool", "pool3s2", "nearest"):
        return np.zeros_like(ref), "exact"
    if kind == "add":
        return np.zeros_like(ref), "f32"
    m = np.abs(x)
    m = np.maximum(np.maximum(m, np.roll(m, 1, 1)), np.roll(m, -1, 1))
    m = np.maximum(np.maximum(m, np.roll(m, 1, 2)), np.roll(m, -1, 2))
    return 2.0 ** -21 * upsample64(m, False), "f32"


def check(dev, ref, e_pre, out, lo=None):
    """Compare a device output with its float64 reference.  Returns a dict:
    worst = max |dev - ref| / (e_pre + rounding of the store), which must be <= 1;
    undecided-rounding misses: where [ref - e_pre, ref + e_pre] holds no fp16 rounding boundary, a correct kernel stores
    exactly fp16(ref) (hi for split outputs); any other value is counted in ``missed``;
    exact = fraction equal to fp16(ref), bias = mean (dev - ref) / ulp16(ref) (fp16 outputs; elements 0 on one side only
    count 0), bias_at = its largest term as (index, device, reference, e_pre, ulps);
    lo_bias (split, reported): mean of sign(lo) (dev - ref) / ulp16(lo) over lo != 0."""
    dev = np.asarray(dev, np.float64)
    bound = e_pre + out_rounding(ref, e_pre, out)
    err = np.abs(dev - ref)
    ratio = err / np.maximum(bound, 2.0 ** -60)
    r = dict(n=int(dev.size), worst=float(ratio.max()) if dev.size else 0.0,
             where=np.unravel_index(int(ratio.argmax()), ratio.shape) if dev.size else None)
    if out in ("f16", "split"):
        hi = dev if out == "f16" else (dev - lo if lo is not None else f16(dev))     # the stored hi plane
        decided = f16(ref - e_pre) == f16(ref + e_pre)
        r["decided"] = float(decided.mean()) if dev.size else 1.0
        r["missed"] = int((decided & (hi != f16(ref))).sum())
        if r["missed"]:
            k = np.argwhere(decided & (hi != f16(ref)))[0]
            r["miss_at"] = (tuple(int(t) for t in k), float(dev[tuple(k)]), float(ref[tuple(k)]), float(e_pre[tuple(k)]))
    if out == "f16":
        r["exact"] = float((dev == f16(ref)).mean()) if dev.size else 1.0
        # An element that is 0 on one side only is a ReLU whose pre-activation lies within e_pre of 0: its error in ulps of
        # a reference of 0 (2^-24) runs to thousands however small, and says nothing about the store's rounding direction;
        # the bound gates it.  So the bias leaves those out.
        u = np.where((dev == 0) == (ref == 0), (dev - ref) / ulp16(ref), 0.0)
        r["bias"] = float(u.mean()) if dev.size else 0.0
        if dev.size:
            k = np.unravel_index(int(np.abs(u).argmax()), u.shape)
            r["bias_at"] = (tuple(int(t) for t in k), float(dev[k]), float(ref[k]), float(e_pre[k]), float(u[k]))
    if out == "split" and lo is not None:
        nz = lo != 0
        r["lo_bias"] = float((np.sign(lo[nz]) * (dev[nz] - ref[nz]) / ulp16(lo[nz])).mean()) if nz.any() else 0.0
        r["lo_n"] = int(nz.sum())
    return r


# ------------------------------------------------------------------------------------------------ float64 primitives
def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x, np.float64)).permute(0, 3, 1, 2)


def _n(t):
    return t.permute(0, 2, 3, 1).contiguous().numpy()


def conv64(x, w, stride, pad_top, pad_left, Hout, Wout):
    """NHWC x (float64), w (k, k, Cin, Cout): zero padding top / left, output Hout x Wout (the bottom / right padding
    follows, negative = rows beyond the last window are unused)."""
    k = w.shape[0]
    B, H, W, C = x.shape
    Hp, Wp = (Hout - 1) * stride + k, (Wout - 1) * stride + k
    xp = np.zeros((B, Hp, Wp, C), np.float64)
    h, ww = min(H, Hp - pad_top), min(W, Wp - pad_left)
    xp[:, pad_top:pad_top + h, pad_left:pad_left + ww] = x[:, :h, :ww]
    wt = torch.from_numpy(np.ascontiguousarray(np.transpose(w, (3, 2, 0, 1)), np.float64))
    with torch.no_grad():
        return _n(F.conv2d(_t(xp), wt, stride=stride))


def tconv64(x, w, k):
    """Conv2DTranspose(k, strides=2, SAME), k = 3 / 4: out[o] += in[i] W[o - 2i + p], p = (k - 2) / 2."""
    B, H, W, C = x.shape
    wt = torch.from_numpy(np.ascontiguousarray(np.transpose(w, (2, 3, 0, 1)), np.float64))
    with torch.no_grad():
        y = F.conv_transpose2d(_t(x), wt, stride=2, padding=(k - 2) // 2)
    return _n(y)[:, :2 * H, :2 * W]


def pool2(x):
    B, H, W, C = x.shape
    return x.reshape(B, H // 2, 2, W // 2, 2, C).max(axis=(2, 4))


def pool3s2(x):
    """ZeroPadding2D(1) + MaxPool2D(3, 2): the padding reads 0."""
    B, H, W, C = x.shape
    xp = np.zeros((B, H + 2, W + 2, C), x.dtype)
    xp[:, 1:-1, 1:-1] = x
    Ho, Wo = H // 2, W // 2
    return np.max(np.stack([xp[:, dy:dy + 2 * Ho:2, dx:dx + 2 * Wo:2] for dy in range(3) for dx in range(3)]), axis=0)


def upsample64(x, bilinear):
    """x2: nearest, or bilinear with half-pixel centres and edge clamp (weights 1/4, 3/4)."""
    if not bilinear:
        return x.repeat(2, axis=1).repeat(2, axis=2)

    def axis(n):
        o = np.arange(2 * n)
        s = (o + 0.5) * 0.5 - 0.5
        f = np.floor(s)
        i0 = np.maximum(f, 0).astype(int)
        i1 = np.minimum(np.ceil(s), n - 1).astype(int)
        return i0, i1, s - f
    B, H, W, C = x.shape
    y0, y1, ly = axis(H)
    x0, x1, lx = axis(W)
    lx = lx[None, None, :, None]
    ly = ly[None, :, None, None]
    tp = x[:, y0][:, :, x0] + (x[:, y0][:, :, x1] - x[:, y0][:, :, x0]) * lx
    bt = x[:, y1][:, :, x0] + (x[:, y1][:, :, x1] - x[:, y1][:, :, x0]) * lx
    return tp + (bt - tp) * ly


def preprocess32(frames, Hnet, Wnet, Cnet, Hres, Wres, mode):
    """k_preprocess replayed in numpy float32: gray <-> rgb, u8 * (1/255), bilinear half-pixel resize, zero padding,
    ImageNet caffe; every step the same correctly rounded fp32 operation as the kernel."""
    f32 = np.float32
    is_u8 = frames.dtype == np.uint8
    B, Hin, Win, Cin = frames.shape
    fr = frames.astype(f32)
    sc = f32(1.0 / 255.0)
    imagenet = mode != ol.PRE_PLAIN
    mode_ch = 0
    if Cin == 3 and (Cnet == 1 or mode == ol.PRE_IMAGENET_CAFFE_GRAY):
        mode_ch = 1
    if Cin == 1 and Cnet == 3:
        mode_ch = 2
    if mode_ch == 1:
        s = sc if is_u8 else f32(1)
        g = (fr[..., 0] * s) * f32(0.2989) + (fr[..., 1] * s) * f32(0.5870)
        g = (g + (fr[..., 2] * s) * f32(0.1140)).astype(f32)
        if is_u8:
            g = (np.trunc(np.clip(g * f32(255.5), 0, 255)).astype(f32) * sc).astype(f32)
        src = np.repeat(g[..., None], Cnet, axis=3)
    else:
        idx = [0 if mode_ch == 2 else ((2 - c) if imagenet else c) for c in range(Cnet)]
        src = fr[..., idx]
        if is_u8:
            src = (src * sc).astype(f32)
    if (Hres, Wres) != (Hin, Win):
        def axis(n_out, n_in):
            scl = f32(n_in) / f32(n_out)
            s = ((np.arange(n_out, dtype=f32) + f32(0.5)) * scl - f32(0.5)).astype(f32)
            fl = np.floor(s)
            return np.maximum(fl, 0).astype(int), np.minimum(np.ceil(s), n_in - 1).astype(int), (s - fl).astype(f32)
        y0, y1, ly = axis(Hres, Hin)
        x0, x1, lx = axis(Wres, Win)
        lx = lx[None, None, :, None]
        ly = ly[None, :, None, None]
        tl, tr = src[:, y0][:, :, x0], src[:, y0][:, :, x1]
        bl, br = src[:, y1][:, :, x0], src[:, y1][:, :, x1]
        tp = (tl + ((tr - tl).astype(f32) * lx).astype(f32)).astype(f32)
        bt = (bl + ((br - bl).astype(f32) * lx).astype(f32)).astype(f32)
        src = (tp + ((bt - tp).astype(f32) * ly).astype(f32)).astype(f32)
    out = np.zeros((B, Hnet, Wnet, Cnet), f32)
    out[:, :Hres, :Wres] = src[:, :Hres, :Wres]
    if imagenet:
        mean = np.asarray([103.939, 116.779, 123.68], f32)
        out = ((out * f32(255)).astype(f32) - mean).astype(f32)
    return out


def net_hw(cm, H, W):
    pre = next(r for r in cm.records if r[0] == ol.PREPROCESS)
    scale = np.frombuffer(np.int32(pre[16]).tobytes(), np.float32)[0]
    Hres, Wres = H, W
    if scale != 1.0:
        Hres, Wres = int(np.float32(H) * scale), int(np.float32(W) * scale)
    ps = max(1, int(pre[17]))
    return -(-Hres // ps) * ps, -(-Wres // ps) * ps, Hres, Wres


# ------------------------------------------------------------------------------------------------ the interpreter
class Audit:
    """One forward pass of a compiled op list.

    ``kinds[i]``: per-op kind of ``sb_model_profile_ops`` (1 tensor core, 2 CUDA core, 0 other); ``conv01``: the fused first
    block ran (``SB_DEBUG`` line "-> fused").  ``precision`` 0, 1 or 2; in precision 1 every buffer is fp32
    (``elem_size`` in sb_model.cu), so it is marked ``f32`` here whatever its record says."""

    def __init__(self, cm, blob, precision, frames, kinds, conv01=False):
        self.cm = cm
        recs = [np.asarray(r) for r in cm.records]
        self.bufs = {int(r[1]): dict(stride=int(r[2]), C=int(r[3]), f32=bool(r[4]) or precision == 1)
                     for r in recs if r[0] == ol.BUFFER}
        self.ops = [r for r in recs if r[0] != ol.BUFFER]
        self.blob = np.asarray(blob, np.float32)
        self.precision = precision
        self.split = precision == 2
        self.frames = frames
        self.kinds = list(kinds)
        self.conv01 = conv01
        B, H, W, Cin = frames.shape
        self.B = B
        self.Hnet, self.Wnet, self.Hres, self.Wres = net_hw(cm, H, W)
        self.pre_i = next(i for i, o in enumerate(self.ops) if o[0] == ol.PREPROCESS)
        self.first_fused = self._first_fusion()
        self.stem_fused = self._stem_fusion()
        self.conv01_ops = self._conv01_ops()
        self.production = True

    # ---- which kernels run (mirrors the input stage's rules in sb_entry.cu: first_fusable, stem_fusable, conv01_fusable,
    # and the fused pool / ADD slots of sb_conv_tc_entry in sb_conv_tc.cu) ----
    def _only_reader(self, buf, reader):
        for j, o in enumerate(self.ops):
            if j == reader or o[0] == ol.PREPROCESS:
                continue
            if o[1] == buf or (o[0] == ol.ADD and o[4] == buf):
                return False
        return True

    def _first_fusion(self):
        if self.precision == 1 or self.pre_i + 1 >= len(self.ops):
            return -1
        pre, cv = self.ops[self.pre_i], self.ops[self.pre_i + 1]
        ib, ob = self.bufs[int(pre[6])], self.bufs[int(cv[6])]
        scale = np.frombuffer(np.int32(pre[16]).tobytes(), np.float32)[0]
        ok = (cv[0] == ol.CONV and cv[1] == pre[6] and cv[9] == 3 and cv[10] == 1 and not cv[11] & ol.F_EXPLICIT_PAD
              and scale == 1.0 and pre[19] == ol.PRE_PLAIN and self.frames.shape[3] == ib["C"] and ib["C"] in (1, 3)
              and cv[3] == ib["C"] and not ob["f32"] and not cv[11] & ol.F_BN and ob["C"] % 8 == 0 and cv[7] % 8 == 0
              and cv[8] in (8, 16, 24, 32, 64) and self._only_reader(int(pre[6]), self.pre_i + 1))
        return self.pre_i + 1 if ok else -1

    def _stem_fusion(self):
        i = self.pre_i + 1
        if self.precision != 0 or self.first_fused >= 0 or i >= len(self.ops):
            return -1
        cv = self.ops[i]
        return i if (cv[0] == ol.CONV and cv[9] == 7 and cv[10] == 2 and self.kinds[i] == 1) else -1

    def _conv01_ops(self):
        c0 = self.first_fused
        if c0 < 0 or self.split or c0 + 2 >= len(self.ops):
            return ()
        a, b = self.ops[c0], self.ops[c0 + 1]
        if b[0] == ol.CONV and b[1] == a[6] and b[18] >= 0 and self.kinds[c0 + 1] == 1 and self._pool_dead(c0 + 1):
            return (c0, c0 + 1)
        return ()

    def _pool_dead(self, i):
        """CONV i runs on the tensor cores, feeds a fused 2x2 pool and nothing else reads its output slice (a CUDA-core
        conv stores its output and the pool runs as its own kernel)."""
        o = self.ops[i]
        if o[0] != ol.CONV or o[18] < 0 or i + 1 >= len(self.ops) or self.ops[i + 1][0] != ol.POOL or not self.ops[i + 1][11] & ol.F_FUSED_POOL:
            return False
        if self.kinds[i] != 1:
            return False
        ext = (3 if self.split else 1) * int(o[8])
        for j, p in enumerate(self.ops):
            if j in (i, i + 1) or p[0] == ol.PREPROCESS:
                continue
            if p[1] == o[6] and p[2] < o[7] + ext and o[7] < p[2] + p[3]:
                return False
            if p[0] == ol.ADD and p[4] == o[6] and p[5] < o[7] + ext and o[7] < p[5] + p[3]:
                return False
        return True

    def _res_fused(self, i):
        o = self.ops[i]
        return (o[0] == ol.CONV and o[11] & ol.F_RESIDUAL and self.kinds[i] == 1 and i + 1 < len(self.ops)
                and self.ops[i + 1][11] & ol.F_FUSED_ADD)

    def internal_buffers(self, production):
        """Buffers a forward must not ask for: the preprocessed frame when the first conv (or stem) reads the frame itself,
        and -- production run -- tensors internal to a fusion (a conv output read only by its fused pool or fused ADD, the
        fused first block's conv0 / conv1 outputs): asking for those switches the forward to separate launches."""
        out = set()
        if self.first_fused >= 0 or self.stem_fused >= 0:
            out.add(int(self.ops[self.pre_i][6]))
        if production:
            for i, o in enumerate(self.ops):
                if self._pool_dead(i) or self._res_fused(i) or i in self.conv01_ops:
                    out.add(int(o[6]))
        return out

    # ---- helpers ----
    def shape(self, b):
        s = self.bufs[b]["stride"]
        return (self.B, self.Hnet // s, self.Wnet // s, self.bufs[b]["C"])

    def engine(self, i):
        if i == (self.conv01_ops or (-1,))[0] and self.conv01 and self.production:
            return "conv01"       # conv0 of k_conv01: fp16 frame and fp16 weights, accumulated by fma on the CUDA cores
        return {1: "tc", 2: "cuda"}.get(self.kinds[i], "tc")

    def out_kind(self, buf):
        if self.bufs[buf]["f32"]:
            return "f32"
        return "split" if self.split else "f16"

    def decode(self, arr, coff, C):
        """Logical values of a slice: split slices are lo + hi (planes C apart, physical 3C)."""
        if not self.split:
            return arr[..., coff:coff + C]
        return arr[..., coff:coff + C] + arr[..., coff + C:coff + 2 * C]

    def decode_err(self, mag):
        """The split elementwise kernels decode lo + hi in fp32 (ld_split): one rounding, 2^-24 relative; 0 otherwise."""
        return 2.0 ** -24 * mag if self.split else np.zeros_like(mag)

    def split_invariants(self, arr, coff, C, name):
        lo, hi, hi2 = (arr[..., coff + p * C:coff + (p + 1) * C] for p in range(3))
        assert np.array_equal(hi, hi2), f"{name}: the two hi planes differ"
        half = 0.5 * ulp16(hi)
        assert np.all(np.abs(lo) <= half), f"{name}: |lo| > ulp(hi) / 2"
        # lo = fp16(v - hi) may round up to exactly ulp(hi) / 2, a tie that fp16(hi + lo) breaks to even
        assert np.array_equal(np.where(np.abs(lo) < half, hi, 0), np.where(np.abs(lo) < half, f16(hi + lo), 0)), \
            f"{name}: hi != fp16(hi + lo)"

    # ---- per-kind references ----
    def _weights(self, op, n_in, fp16w):
        k = int(op[9])
        w = self.blob[int(op[12]):int(op[12]) + k * k * n_in * int(op[8])].reshape(k, k, n_in, int(op[8]))
        w = f16(w) if fp16w else w.astype(np.float64)
        b = self.blob[int(op[13]):int(op[13]) + int(op[8])].astype(np.float64) if op[13] >= 0 else np.zeros(int(op[8]))
        return w, b

    def conv(self, i, x, e_in=None, res=None, relu=None):
        """Reference of CONV / TCONV op i on physical input x -> (value after the epilogue, e_pre, n_steps)."""
        op = self.ops[i]
        k, st = int(op[9]), int(op[10])
        eng = self.engine(i)
        w, b = self._weights(op, x.shape[3], eng in ("tc", "conv01"))
        ob = self.shape(int(op[6]))
        if op[0] == ol.TCONV:
            s, A = tconv64(x, w, k), tconv64(np.abs(x), np.abs(w), k)
            prop = tconv64(e_in, np.abs(w), k) if e_in is not None else 0.0
            taps = ((k + 1) // 2) ** 2
        else:
            Hin, Win = x.shape[1:3]
            if op[11] & ol.F_EXPLICIT_PAD:
                pt, pl = int(op[16]), int(op[17])
            else:
                pt = max((ob[1] - 1) * st + k - Hin, 0) // 2
                pl = max((ob[2] - 1) * st + k - Win, 0) // 2
            s = conv64(x, w, st, pt, pl, ob[1], ob[2])
            A = conv64(np.abs(x), np.abs(w), st, pt, pl, ob[1], ob[2])
            prop = conv64(e_in, np.abs(w), st, pt, pl, ob[1], ob[2]) if e_in is not None else 0.0
            taps = k * k
        n = taps * (math.ceil(x.shape[3] / 16) if eng == "tc" else x.shape[3])      # K = 16 steps, or one fma per product
        v = s + b
        mag = np.abs(s) + np.abs(b)
        if res is not None:
            v = v + res
            mag = mag + np.abs(res)
        if relu is None:
            relu = bool(op[11] & ol.F_RELU)
        if relu:
            v = np.maximum(v, 0)
        sc = sh = None
        if op[11] & ol.F_BN:
            sc = self.blob[int(op[14]):int(op[14]) + int(op[8])].astype(np.float64)
            sh = self.blob[int(op[15]):int(op[15]) + int(op[8])].astype(np.float64)
            e = elem_bound(A, mag, n, prop, sc, np.abs(v * sc) + np.abs(sh))
            v = v * sc + sh
        else:
            e = elem_bound(A, mag, n, prop)
        return v, e, n

    # ---- the audit ----
    def run(self, dev, production):
        """dev: {buffer id: float array of the whole buffer} from one forward (fp16 buffers as float32).  Returns one row
        per checked output: dict(op, what, engine, n, worst, exact, bias, missed, ...)."""
        self.production = production     # k_conv01 runs only when no tensor internal to it is fetched
        rows = []
        chain = {}                      # buffer id -> (value, e incl. its fp16 rounding) of a tensor that is not visible
        pending = {}                    # conv op -> (value, e_pre) checked through its fused pool / ADD
        internal = self.internal_buffers(production)
        pre32 = None
        for i, op in enumerate(self.ops):
            kind = int(op[0])
            ob = int(op[6])
            if kind == ol.PREPROCESS:
                C = self.bufs[ob]["C"]
                pre32 = preprocess32(self.frames, self.Hnet, self.Wnet, C, self.Hres, self.Wres, int(op[19]))
                if ob in internal:
                    continue
                ref = pre32.astype(np.float64)
                if self.split and not self.bufs[ob]["f32"]:
                    raise AssertionError("precision 2 keeps the preprocessed frame in fp32")
                rows.append(self._row(i, "preprocess", dev[ob][..., :C], None, ref, np.zeros_like(ref), self.out_kind(ob)))
                continue
            if kind in (ol.CONV, ol.TCONV):
                ib, coff, cin = int(op[1]), int(op[2]), int(op[3])
                e_in = None
                if ib == int(self.ops[self.pre_i][6]) and ib in internal:
                    x = pre32[..., coff:coff + cin].astype(np.float64)
                    if self.engine(i) in ("tc", "conv01"):
                        x = f16(x)
                elif ib in chain:
                    x, e_in = chain[ib]
                    x, e_in = x[..., coff:coff + cin], e_in[..., coff:coff + cin]
                else:
                    x = dev[ib][..., coff:coff + cin].astype(np.float64)
                res, relu, dst = None, None, (ob, int(op[7]))
                fused_add = production and self._res_fused(i)
                if fused_add:
                    rb, rc = int(op[20]), int(op[21])
                    res = self.decode(dev[rb].astype(np.float64), rc, int(op[8]))
                    relu = bool(self.ops[i + 1][11] & ol.F_RELU)
                    dst = (int(op[22]), int(op[23]))
                v, e, n = self.conv(i, x, e_in, res, relu)
                what = ("tconv" if kind == ol.TCONV else f"conv{int(op[9])}x{int(op[9])}/{int(op[10])}") + \
                       (" +res" if fused_add else "") + (" +bn" if op[11] & ol.F_BN else "")
                if ob in internal and not fused_add:
                    if self.conv01_ops and i == self.conv01_ops[0]:
                        chain[ob] = (self._place(ob, int(op[7]), v), self._place(ob, int(op[7]), e + 0.5 * ulp16(np.abs(v) + e)))
                    elif self._pool_dead(i):
                        pending[i] = (v, e)
                    else:
                        raise AssertionError(f"op {i} writes buffer {ob}, which this run does not fetch, and nothing checks it")
                    continue
                rows.append(self._row(i, what, *self._slice(dev, dst[0], dst[1], int(op[8])), v, e, self.out_kind(dst[0]),
                                      engine=self.engine(i), steps=n))
                continue
            if kind == ol.POOL:
                C = int(op[3]) // (3 if self.split else 1)
                prod = i - 1
                if prod in pending and self.ops[prod][6] == op[1]:
                    # fp16: max of the rounded values = fp16(max of the unrounded ones) (rounding is monotonic); precision
                    # 2 pools the fp32 values before the split.  Either way one store rounding of a value within
                    # max(e) of the reference, which check() adds
                    v, e = pending.pop(prod)
                    ok = self.out_kind(ob)
                    ref = pool2(v) if op[9] != 3 else pool3s2(v)
                    ep = pool2(e) if op[9] != 3 else pool3s2(e)
                    rows.append(self._row(i, "pool(conv)", *self._slice(dev, ob, int(op[7]), C), ref, ep, ok,
                                          engine=self.engine(prod)))
                    continue
                x = self.decode(dev[int(op[1])].astype(np.float64), int(op[2]), C)
                ref = pool3s2(x) if op[9] == 3 else pool2(x)
                e, ok = (self.decode_err(np.abs(ref)), self.out_kind(ob)) if self.precision != 1 else elementwise_bound("pool", ref)
                rows.append(self._row(i, "pool3s2" if op[9] == 3 else "pool2", *self._slice(dev, ob, int(op[7]), C), ref, e, ok))
                continue
            if kind == ol.UPSAMPLE:
                C = int(op[3]) // (3 if self.split else 1)
                x = self.decode(dev[int(op[1])].astype(np.float64), int(op[2]), C)
                bil = bool(op[11] & ol.F_BILINEAR)
                ref = upsample64(x, bil)
                if self.precision == 1:
                    e, ok = elementwise_bound("bilinear" if bil else "nearest", ref, x)
                else:
                    e = np.zeros_like(ref)
                    if bil:                    # three fp32 lerps: a few roundings of the largest of the four corners
                        m = np.abs(x)
                        m = np.maximum(np.maximum(m, np.roll(m, 1, 1)), np.roll(m, -1, 1))
                        m = np.maximum(np.maximum(m, np.roll(m, 1, 2)), np.roll(m, -1, 2))
                        e = 2.0 ** -21 * upsample64(m, False)
                    e = e + self.decode_err(upsample64(np.abs(x), False) if not bil else upsample64(m, False))
                    ok = self.out_kind(ob)
                rows.append(self._row(i, "upsample-" + ("bilinear" if bil else "nearest"), *self._slice(dev, ob, int(op[7]), C),
                                      ref, e, ok))
                continue
            if kind == ol.ADD:
                if production and i > 0 and self._res_fused(i - 1):
                    continue                                  # checked as the residual epilogue of the conv before it
                C = int(op[3]) // (3 if self.split else 1)
                a = self.decode(dev[int(op[1])].astype(np.float64), int(op[2]), C)
                b = self.decode(dev[int(op[4])].astype(np.float64), int(op[5]), C)
                ref = a + b
                e = 2.0 ** -24 * (np.abs(a) + np.abs(b)) + self.decode_err(np.abs(a) + np.abs(b))
                if op[11] & ol.F_RELU:
                    ref = np.maximum(ref, 0)
                ok = self.out_kind(ob)
                if self.precision == 1:
                    e, ok = elementwise_bound("add", ref)
                rows.append(self._row(i, "add", *self._slice(dev, ob, int(op[7]), C), ref, e, ok))
                continue
            if kind == ol.COPY:
                C = int(op[3])
                ref = dev[int(op[1])][..., int(op[2]):int(op[2]) + C].astype(np.float64)
                got = dev[ob][..., int(op[7]):int(op[7]) + C].astype(np.float64)
                rows.append(dict(op=i, what="copy", engine="", n=int(got.size), worst=0.0 if np.array_equal(got, ref) else np.inf))
                continue
        assert not pending, f"conv ops {sorted(pending)} have a fused pool that was never checked"
        return rows

    def _place(self, buf, coff, v):
        full = np.zeros(self.shape(buf), np.float64)
        full[..., coff:coff + v.shape[3]] = v
        return full

    def _slice(self, dev, buf, coff, C):
        """(device logical values, lo plane or None) of an output slice; split slices have their invariants checked."""
        a = dev[buf].astype(np.float64)
        if self.split and not self.bufs[buf]["f32"]:
            self.split_invariants(a, coff, C, f"buffer {buf} [{coff}:{coff + 3 * C}]")
            return self.decode(a, coff, C), a[..., coff:coff + C]
        return a[..., coff:coff + C], None

    def _row(self, i, what, got, lo, ref, e, out, engine="", steps=0):
        r = check(got, ref, e, out, lo)
        r.update(op=i, what=what, engine=engine, steps=steps, out=out)
        return r


def store(aud, arr, buf, coff, v, mode):
    """Write logical values v into a buffer slice.  mode 'exact': float64 as is (split: hi = fp16(v), lo = v - hi
    unrounded); 'device': fp16 round to nearest / the split store / fp32."""
    C = v.shape[3]
    if aud.bufs[buf]["f32"]:
        arr[..., coff:coff + C] = v if mode == "exact" else v.astype(np.float32)
    elif aud.split:
        hi = f16(v)
        lo = v - hi if mode == "exact" else f16(v - hi)
        arr[..., coff:coff + C], arr[..., coff + C:coff + 2 * C], arr[..., coff + 2 * C:coff + 3 * C] = lo, hi, hi
    else:
        arr[..., coff:coff + C] = v if mode == "exact" else f16(v)


def interpret(aud, mode="exact", production=False, conv_fn=None):
    """Chain the float64 references on their own outputs from the frame: {buffer id: array}.  ``conv_fn(aud, i, x, res,
    relu)`` replaces the float64 conv (e.g. by an emulation of the device's accumulation); ``production`` runs a fused
    residual ADD in the conv's epilogue, as the tensor-core path does."""
    buf = {b: np.zeros(aud.shape(b), np.float64) for b in aud.bufs}
    conv = conv_fn or (lambda a, i, x, res, relu: a.conv(i, x, None, res, relu)[0])
    for i, op in enumerate(aud.ops):
        kind, ob = int(op[0]), int(op[6])
        if kind == ol.PREPROCESS:
            C = aud.bufs[ob]["C"]
            buf[ob][..., :C] = preprocess32(aud.frames, aud.Hnet, aud.Wnet, C, aud.Hres, aud.Wres, int(op[19]))
            if not aud.bufs[ob]["f32"] and mode != "exact":
                buf[ob] = f16(buf[ob])
        elif kind in (ol.CONV, ol.TCONV):
            x = buf[int(op[1])][..., int(op[2]):int(op[2]) + int(op[3])]
            if production and aud._res_fused(i):
                res = aud.decode(buf[int(op[20])], int(op[21]), int(op[8]))
                v = conv(aud, i, x, res, bool(aud.ops[i + 1][11] & ol.F_RELU))
                store(aud, buf[int(op[22])], int(op[22]), int(op[23]), v, mode)
            else:
                store(aud, buf[ob], ob, int(op[7]), conv(aud, i, x, None, None), mode)
        elif kind == ol.ADD and production and aud._res_fused(i - 1):
            continue
        elif kind in (ol.POOL, ol.UPSAMPLE, ol.ADD):
            C = int(op[3]) // (3 if aud.split else 1)
            x = aud.decode(buf[int(op[1])], int(op[2]), C)
            if kind == ol.POOL:
                v = pool3s2(x) if op[9] == 3 else pool2(x)
            elif kind == ol.UPSAMPLE:
                v = upsample64(x, bool(op[11] & ol.F_BILINEAR))
            else:
                v = x + aud.decode(buf[int(op[4])], int(op[5]), C)
                if op[11] & ol.F_RELU:
                    v = np.maximum(v, 0)
            store(aud, buf[ob], ob, int(op[7]), v, mode)
        elif kind == ol.COPY:
            buf[ob][..., int(op[7]):int(op[7]) + int(op[3])] = buf[int(op[1])][..., int(op[2]):int(op[2]) + int(op[3])]
    return buf


def synthetic_weights(cm, seed):
    """Synthetic weights with non-trivial biases and BN statistics, so that every epilogue term is exercised; the last BN
    of each residual branch is scaled down so that 16 ResNet blocks of He-normal weights stay well inside fp16."""
    from sleap_b200.nn import architectures as A
    w = A.make_synthetic_weights(cm, seed)
    rng = np.random.default_rng(seed + 1)
    for L in cm.layers:
        if L["kind"] in ("conv", "tconv"):
            w[L["name"]]["bias"] = rng.normal(0, 0.1, size=L["cout"]).astype(np.float32)
        else:
            c = L["c"]
            g = 0.3 if L["name"].endswith("_3_bn") else 1.0
            w[L["name"]] = dict(gamma=(g * rng.uniform(0.5, 1.5, c)).astype(np.float32), beta=rng.normal(0, 0.1, c).astype(np.float32),
                                mean=rng.normal(0, 0.1, c).astype(np.float32), var=rng.uniform(0.5, 1.5, c).astype(np.float32))
    return w


def format_rows(rows, forms=None):
    lines = [f"{'op':>4} {'what':<22} {'eng':<5} {'form':<10} {'n':>10} {'worst':>7} {'decided':>8} {'missed':>6} "
             f"{'exact':>7} {'bias/ulp':>9} {'lo_bias':>8}"]
    for r in rows:
        f = ",".join(sorted((forms or {}).get(r["op"], ())))
        lines.append(f"{r['op']:>4} {r['what']:<22} {r['engine']:<5} {f:<10} {r['n']:>10} {r['worst']:>7.3f} "
                     f"{r.get('decided', float('nan')):>8.4f} {r.get('missed', 0):>6} {r.get('exact', float('nan')):>7.4f} "
                     f"{r.get('bias', float('nan')):>9.4f} {r.get('lo_bias', float('nan')):>8.4f}")
    return "\n".join(lines)
