"""Achieved HBM bandwidth of each memory-bound row-kernel class of the bench.py default workload, against the HBM
floor.

    python bench.py --gpus 1 > bench.json
    python tools/row_rates.py bench.json          # or: ... | python tools/row_rates.py -

The per-class times are bench.py's kernel_time_shares (one CUDA event pair per launch).  The bytes are those each
kernel has to move through HBM at the default workload's shapes: 64 x 30 s clips = 128 chunks of L = 1500 frames,
final0 (D = 512, 6 main layers; frontend blocks at C = 32, 64, 128 over F = 32, 16, 8 frequency planes; head_dim 32).
Weights are read once per CTA and stay in L2, so they are not counted.  The floor is bytes over the HBM bandwidth of
MEASURED_PEAKS.json ("hbm_gbs", as bench.py reads it) when that file is present, otherwise the 3.35 TB/s of NVIDIA's H100 SXM data sheet.
"""
import argparse
import json
import os
import sys

ROWS = 128 * 1500  # frames per step: one row per frame in the main layers
DATASHEET_TBPS = 3.35

# class -> list of (launches per step, rows per launch, HBM bytes per row)
#   qkv_fused: 4C fp32 x in; 6C 16-bit q, k, v out; 4 per head fp32 gate out
#   ff_fused:  4C fp32 x in, 2C 16-bit O in (attention out-projection fused in front), 4C fp32 x out; the FFN in front
#              of each convolution also writes a 2C 16-bit copy of its result
#   attn_freq: 6C 16-bit q, k, v in, 4 per head gates in, 2C 16-bit O out
#   norm, norm_front: 4C fp32 in, 2C 16-bit out
#   stem: one 128-bin fp32 spectrogram frame in, 32 planes x 32 channels fp32 out
CLASSES = {
    "qkv_fused_c32": [(2, 32 * ROWS, 4 * 32 + 6 * 32 + 4 * 1)],
    "qkv_fused_c64": [(2, 16 * ROWS, 4 * 64 + 6 * 64 + 4 * 2)],
    "ff_fused_c32": [(1, 32 * ROWS, 4 * 32 + 2 * 32 + 4 * 32), (1, 32 * ROWS, 4 * 32 + 2 * 32 + 4 * 32 + 2 * 32)],
    "ff_fused_c64": [(1, 16 * ROWS, 4 * 64 + 2 * 64 + 4 * 64), (1, 16 * ROWS, 4 * 64 + 2 * 64 + 4 * 64 + 2 * 64)],
    "attn_freq": [(1, 32 * ROWS, 6 * 32 + 4 * 1 + 2 * 32), (1, 16 * ROWS, 6 * 64 + 4 * 2 + 2 * 64),
                  (1, 8 * ROWS, 6 * 128 + 4 * 4 + 2 * 128)],
    "norm": [(12, ROWS, 4 * 512 + 2 * 512)],
    "norm_front": [(4, 8 * ROWS, 4 * 128 + 2 * 128)],
    "stem": [(1, ROWS, 4 * 128 + 4 * 32 * 32)],
}
FUSED = ("qkv_fused_c32", "qkv_fused_c64", "ff_fused_c32", "ff_fused_c64")


def gbytes(terms):
    return sum(n * rows * b for n, rows, b in terms) / 1e9


def hbm_peak(root):
    path = os.path.join(root, "MEASURED_PEAKS.json")
    if os.path.exists(path):
        with open(path) as f:
            peaks = json.load(f)
        if "hbm_gbs" in peaks:
            return float(peaks["hbm_gbs"]) / 1e3, "MEASURED_PEAKS.json hbm_gbs (measured)"
    return DATASHEET_TBPS, "H100 SXM data sheet (not measured)"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("bench_json", help="file holding bench.py's JSON line (the last line that parses), or - for stdin")
    args = ap.parse_args()
    text = sys.stdin.read() if args.bench_json == "-" else open(args.bench_json).read()
    line = None
    for raw in text.splitlines():
        raw = raw.strip()
        if raw.startswith("{"):
            try:
                cand = json.loads(raw)
            except json.JSONDecodeError:
                continue
            if "kernel_time_shares" in cand:
                line = cand
    if line is None:
        sys.exit("no bench.py JSON line with kernel_time_shares found")
    # CLASSES holds the shapes of the default workload only
    cfg = line.get("config", {})
    wl = cfg.get("workload", "")
    if cfg.get("batch_per_gpu") != 64 or "(128 chunks of 1500 frames" not in wl or "final0" not in wl:
        sys.exit("the bench line is not the default workload (final0, 64 x 30 s clips = 128 chunks of 1500 frames); "
                 "the row counts in this tool would not match it")
    shares = line["kernel_time_shares"]
    tbps, src = hbm_peak(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    rows = []
    for name, terms in CLASSES.items():
        gb = gbytes(terms)
        ms = shares.get(name, {}).get("ms_per_step")
        floor_ms = gb / tbps  # GB / (TB/s) = ms
        rows.append({"class": name, "gb_per_step": round(gb, 3), "ms_per_step": ms,
                     "gbps": round(gb / (ms / 1e3), 1) if ms else None, "floor_ms": round(floor_ms, 3),
                     "x_floor": round(ms / floor_ms, 2) if ms else None})
    fused = [r for r in rows if r["class"] in FUSED]
    f_ms = sum(r["ms_per_step"] or 0.0 for r in fused)
    f_floor = sum(r["floor_ms"] for r in fused)
    print(f"HBM floor at {tbps} TB/s: {src}")
    print(f"{'class':<16}{'GB':>8}{'ms':>9}{'GB/s':>9}{'floor ms':>10}{'x floor':>9}")
    fmt = lambda v, w, p: f"{v:>{w}.{p}f}" if v is not None else f"{'-':>{w}}"
    for r in rows:
        print(f"{r['class']:<16}{fmt(r['gb_per_step'], 8, 3)}{fmt(r['ms_per_step'], 9, 3)}{fmt(r['gbps'], 9, 1)}"
              f"{fmt(r['floor_ms'], 10, 3)}{fmt(r['x_floor'], 9, 2)}")
    print(f"{'fused (4)':<16}{sum(r['gb_per_step'] for r in fused):>8.3f}{f_ms:>9.3f}{'':>9}{f_floor:>10.3f}"
          f"{(f_ms / f_floor if f_ms else 0.0):>9.2f}")
    print(json.dumps({"bench_value": line.get("value"), "hbm_tbps": tbps, "hbm_source": src, "rows": rows,
                      "fused_ms_per_step": round(f_ms, 3), "fused_floor_ms": round(f_floor, 3)}))


if __name__ == "__main__":
    main()
