"""Algorithmic TFLOP/s of each GEMM class of the bench.py default workload, next to torch.matmul (cuBLAS) at the
same shapes on the same card.

    python bench.py --gpus 1 > bench.json
    python tools/gemm_rates.py bench.json          # or: ... | python tools/gemm_rates.py -

The per-class times are bench.py's kernel_time_shares (one CUDA event pair per launch).  The shapes are those of the
default workload: 64 x 30 s clips = 128 chunks of L = 1500 frames, final0 (D = 512, 6 main layers, frontend block 2
at C = 128 over F = 8 frequency planes).  Work is 2 M N K per launch.  The yardstick times torch.matmul of a
[M, K] x [K, N] fp16 product with fp32 accumulation (reduced-precision reductions off) with CUDA events.
"""
import argparse
import json
import sys

M_MAIN = 128 * 1500       # main layers: one row per frame
M_FRONT = 128 * 1500 * 8  # frontend block 2: one row per (frame, frequency plane)

# class -> list of (launches per step, M, N, K)
CLASSES = {
    "gemm_qkv": [(6, M_MAIN, 1536, 512)],
    "gemm_ff1": [(6, M_MAIN, 2048, 512)],
    "gemm_ff2": [(6, M_MAIN, 512, 2048)],
    "gemm_attn_out": [(6, M_MAIN, 512, 512)],
    "gemm_qkv_front": [(2, M_FRONT, 384, 128)],
    "gemm_ff1_front": [(2, M_FRONT, 512, 128)],
    "gemm_ff2_front": [(2, M_FRONT, 128, 512)],
    "gemm_attn_out_front": [(2, M_FRONT, 128, 128)],
    "gemm_conv": [(1, 2 * M_FRONT, 64, 6 * 32), (1, M_FRONT, 128, 6 * 64), (1, M_FRONT // 2, 256, 6 * 128)],
    "gemm_frontend_linear": [(1, M_MAIN, 512, 4 * 256)],
}


def tflop(shapes):
    return sum(2.0 * n * m * nn * k for n, m, nn, k in shapes) / 1e12


def matmul_ms(m, n, k, reps=20):
    import torch

    a = torch.randn(m, k, device="cuda", dtype=torch.float16)
    b = torch.randn(k, n, device="cuda", dtype=torch.float16)
    for _ in range(3):
        torch.matmul(a, b)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        torch.matmul(a, b)
    e1.record()
    torch.cuda.synchronize()
    del a, b
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("bench_json", help="file holding bench.py's JSON line (the last line that parses), or - for stdin")
    ap.add_argument("--no-cublas", action="store_true", help="skip the torch.matmul yardstick (no GPU needed)")
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
                 "the GEMM shapes in this tool would not match it")
    shares = line["kernel_time_shares"]
    gpu = ""
    if not args.no_cublas:
        import torch

        torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction = False
        gpu = torch.cuda.get_device_name(0)
    rows = []
    for name, shapes in CLASSES.items():
        ms = shares.get(name, {}).get("ms_per_step")
        tf = tflop(shapes)
        ours = tf / (ms / 1e3) if ms else None
        ref_ms = None if args.no_cublas else sum(n * matmul_ms(m, nn, k) for n, m, nn, k in shapes)
        ref = tf / (ref_ms / 1e3) if ref_ms else None
        rows.append({"class": name, "tflop_per_step": round(tf, 3), "ms_per_step": ms,
                     "tflops": round(ours, 1) if ours else None,
                     "cublas_ms_per_step": round(ref_ms, 3) if ref_ms else None,
                     "cublas_tflops": round(ref, 1) if ref else None,
                     "frac_of_cublas": round(ours / ref, 3) if ours and ref else None})
    print(f"{'class':<22}{'TFLOP':>8}{'ms':>9}{'TFLOP/s':>9}{'cuBLAS ms':>11}{'cuBLAS TFLOP/s':>16}{'ratio':>7}")
    fmt = lambda v, w, p: f"{v:>{w}.{p}f}" if v is not None else f"{'-':>{w}}"
    for r in rows:
        print(f"{r['class']:<22}{fmt(r['tflop_per_step'], 8, 3)}{fmt(r['ms_per_step'], 9, 3)}{fmt(r['tflops'], 9, 1)}"
              f"{fmt(r['cublas_ms_per_step'], 11, 3)}{fmt(r['cublas_tflops'], 16, 1)}{fmt(r['frac_of_cublas'], 7, 3)}")
    print(json.dumps({"gpu": gpu, "bench_value": line.get("value"), "rows": rows}))


if __name__ == "__main__":
    main()
