"""Per-layer floors of the C4 network (8 frames of 1024x1024) next to the measured per-op times.

  BENCH_VERBOSE=1 python bench.py 2> per_op.txt; python tools/layer_rooflines.py per_op.txt floors.md [L2_TBS]

Floors: tensor = algorithmic FLOPs / 989 TFLOP/s (H100 SXM data sheet, dense fp16, 700 W);
HBM = (activations in + out (+ fused pool output) at their storage width) / 3.35 TB/s (H100 SXM data sheet).
`MEASURED_PEAKS.json` at the repository root (`bf16_tflops`, `hbm_gbs`), when present, replaces both figures, as in
bench.py.  The bound of a layer is the larger floor.
L2 columns (3x3 convs and k3 transposed convs only): the bytes the streaming form of k_conv_wg pulls from L2 into the SMs
(every 128-pixel CTA loads its activation boxes and its whole weight slice), and, given an L2 read rate in TB/s
(`tools/bw_probe.py`, "L2-resident"), the time that traffic takes at that rate; then the same for the wide form
k_conv_wg_hw (3x3 convs) or the fused transposed-conv form k_tconv_wg_hw (k3 transposed convs) where it is eligible.
"""
import json
import os
import re
import sys

B = 8


def _peaks():
    p = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return float(d["bf16_tflops"]), float(d["hbm_gbs"]) / 1e3, "MEASURED_PEAKS.json"
    return 989.0, 3.35, "H100 SXM data sheet (700 W)"


PEAK_TF, PEAK_TBS, PEAK_SRC = _peaks()
# (op index in the per-op table, name, Cin, Cout, input grid H(=W), output grid, taps, pooled copy, out bytes/elem)
LAYERS = [
    (1, "conv 1->16 (Toeplitz view)", 1, 16, 1024, 1024, 9, False, 2),
    (2, "conv 16->16 + pool", 16, 16, 1024, 1024, 9, True, 2),
    (4, "conv 16->32", 16, 32, 512, 512, 9, False, 2),
    (5, "conv 32->32 + pool", 32, 32, 512, 512, 9, True, 2),
    (7, "conv 32->64", 32, 64, 256, 256, 9, False, 2),
    (8, "conv 64->64 + pool", 64, 64, 256, 256, 9, True, 2),
    (10, "conv 64->128", 64, 128, 128, 128, 9, False, 2),
    (11, "conv 128->128 + pool", 128, 128, 128, 128, 9, True, 2),
    (13, "conv 128->256", 128, 256, 64, 64, 9, False, 2),
    (14, "conv 256->256 + pool", 256, 256, 64, 64, 9, True, 2),
    (16, "conv 256->512 (middle)", 256, 512, 32, 32, 9, False, 2),
    (17, "conv 512->512 (middle)", 512, 512, 32, 32, 9, False, 2),
    (18, "tconv 512->256 (32->64)", 512, 256, 32, 64, 2.25, False, 2),
    (19, "conv 512->256", 512, 256, 64, 64, 9, False, 2),
    (20, "conv 256->256", 256, 256, 64, 64, 9, False, 2),
    (21, "tconv 256->128 (64->128)", 256, 128, 64, 128, 2.25, False, 2),
    (22, "conv 256->128", 256, 128, 128, 128, 9, False, 2),
    (23, "conv 128->128", 128, 128, 128, 128, 9, False, 2),
    (24, "tconv 128->64 (128->256)", 128, 64, 128, 256, 2.25, False, 2),
    (25, "conv 128->64", 128, 64, 256, 256, 9, False, 2),
    (26, "conv 64->64", 64, 64, 256, 256, 9, False, 2),
    (27, "head 1x1 64->13 (fp32 out)", 64, 13, 256, 256, 1, False, 4),
    (28, "head 1x1 128->24 (fp32 out)", 128, 24, 128, 128, 1, False, 4),
]


def _wg_n(n):
    for c in (16, 32, 48, 64, 96, 128, 192):
        if n <= c:
            return c
    return 256


def l2_bytes_streaming(cin, cout, hin, taps):
    """Bytes the streaming k_conv_wg moves from L2 into shared memory for one layer of B frames (None: not modelled)."""
    kc = 64 if cin > 32 else (32 if cin > 16 else 16)
    chunks = -(-cin // kc)
    cp = -(-cout // 16) * 16
    n = _wg_n(min(cp, 256))
    n_tiles = -(-cp // n)
    tiles = -(-hin // 16) * -(-hin // 8)
    if taps == 9:                # 3 filter columns: one 10-row box each, 9 weight slices
        rows, slices = 3 * 10, 9
    elif taps == 2.25:           # k3 transposed conv, 4 phases over the input grid: 3 + 3 boxes of 9 / 8 rows, 9 slices
        rows, slices = 3 * 9 + 3 * 8, 9
    else:
        return None
    return B * tiles * n_tiles * chunks * (rows * 16 * kc * 2 + slices * n * kc * 2)


def l2_bytes_wide(cin, cout, hin, taps):
    """The same for the wide form k_conv_wg_hw (3x3 convs with C_in > 32; None: not eligible): per item (16 x 8 by pixels,
    one N tile of n <= 128 channels) and 64-channel chunk, one (8 by + 2) x 18-pixel halo patch and 9 weight slices.
    For a k3 transposed conv, the fused form k_tconv_wg_hw: per 16 x 16 input tile, N tile and 64-channel chunk, the four
    phases load 2 + 1 + 2 + 1 activation boxes of 17 x 16 pixels and 4 + 2 + 2 + 1 weight slices."""
    if taps not in (9, 2.25) or cin <= 32:
        return None
    n = min(_wg_n(-(-cout // 16) * 16), 128)
    if cout % n:
        return None
    if taps == 2.25:
        tiles = (-(-hin // 16)) ** 2
        return B * tiles * (cout // n) * -(-cin // 64) * (6 * 17 * 16 * 64 * 2 + 9 * n * 64 * 2)
    by = 4 if n <= 64 else 2
    items = -(-hin // 16) * -(-hin // (8 * by))
    return B * items * (cout // n) * -(-cin // 64) * ((8 * by + 2) * 18 * 64 * 2 + 9 * n * 64 * 2)


def main(src, out, l2_tbs=None):
    ms = {}
    for line in open(src):
        m = re.match(r"\[op\s*(\d+)\] kind=\d+\s+([\d.]+) us", line)
        if m:
            ms[int(m.group(1))] = float(m.group(2))
    rows = ["| op | layer | measured us | GFLOP | tensor floor us | bytes MB | HBM floor us | bound | floor / measured | L2 GB (streaming) | L2 us "
            "| L2 GB (wide / fused tconv) | L2 us (wide / fused tconv) |",
            "|---|---|---|---|---|---|---|---|---|---|---|---|---|"]
    tot_m = tot_f = tot_l2 = 0.0

    def l2_cols(b):
        if b is None:
            return "| | |"
        return f"| {b / 1e9:.2f} | " + (f"{b / (l2_tbs * 1e12) * 1e6:.1f} |" if l2_tbs else "|")
    layers = list(LAYERS)
    if ms.get(2, 1e9) < 10.0:        # fused first block (k_conv01): op 1 holds both convs + the pool, op 2 is an empty slot
        flops = sum(2.0 * 9 * ci * co * 1024 * 1024 * B for ci, co in ((1, 16), (16, 16)))
        t_tensor = flops / (PEAK_TF * 1e12) * 1e6
        byts = B * 1024 * 1024 * 1 + B * 512 * 512 * 16 * 2          # uint8 frames in, pooled fp16 out: nothing else leaves the SM
        t_hbm = byts / (PEAK_TBS * 1e12) * 1e6
        meas = ms[1] + ms[2]
        floor = max(t_tensor, t_hbm)
        tot_m += meas
        tot_f += floor
        rows.append(f"| 1+2 | fused first block 1->16->16 + pool (k_conv01) @1024² | {meas:.1f} | {flops / 1e9:.2f} | {t_tensor:.1f} | {byts / 1e6:.1f} | "
                    f"{t_hbm:.1f} | {'tensor' if t_tensor >= t_hbm else 'HBM'} | {floor / meas:.2f} | | | | |")
        layers = [l for l in layers if l[0] not in (1, 2)]
    for op, name, cin, cout, hin, hout, taps, pool, ob in layers:
        flops = 2.0 * taps * cin * cout * hout * hout * B
        t_tensor = flops / (PEAK_TF * 1e12) * 1e6
        in_b = B * hin * hin * cin * (1 if cin == 1 else 2)
        out_b = B * hout * hout * cout * ob * (1.25 if pool else 1.0)
        t_hbm = (in_b + out_b) / (PEAK_TBS * 1e12) * 1e6
        floor = max(t_tensor, t_hbm)
        meas = ms.get(op, float("nan"))
        tot_m += meas
        tot_f += floor
        l2b = None if op == 1 else l2_bytes_streaming(cin, cout, hin, taps)
        tot_l2 += l2b or 0.0
        rows.append(f"| {op} | {name} @{hin}² | {meas:.1f} | {flops / 1e9:.2f} | {t_tensor:.1f} | {(in_b + out_b) / 1e6:.1f} | {t_hbm:.1f} | "
                    f"{'tensor' if t_tensor >= t_hbm else 'HBM'} | {floor / meas:.2f} " + l2_cols(l2b) + l2_cols(l2_bytes_wide(cin, cout, hin, taps))[1:])
    rows.append(f"| | **all conv layers** | **{tot_m:.1f}** | | | | | | **{tot_f / tot_m:.2f}** (sum of floors {tot_f:.1f} us) | "
                f"**{tot_l2 / 1e9:.2f}** | " + (f"**{tot_l2 / (l2_tbs * 1e12) * 1e6:.1f}** |" if l2_tbs else "|") + " | |")
    text = ("# C4 per-layer floors vs measured (8 frames, one H100)\n\nMeasured: CUDA-event per-op times of `bench.py` (`sb_model_profile_ops`), file `" + src +
            f"`.  Floors: {PEAK_TF:.0f} TFLOP/s and {PEAK_TBS:.2f} TB/s ({PEAK_SRC}); see tools/layer_rooflines.py.\n\n" + "\n".join(rows) + "\n")
    open(out, "w").write(text)
    print(text)


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2], float(sys.argv[3]) if len(sys.argv) > 3 else None)
