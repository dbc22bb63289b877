"""Per-kernel times of the parity mode's split-operand Gram and residual update at the block fit's shapes (GPU box).

    python tools/split_pair_times.py [--rows 1048576] [--block 4096] [--classes 1000] [--iters 5]

Imports keystone_b200 from the current directory, so running it from another checkout times that build.  One JSON line per kernel:
  gram_g   the G-Gram launch (S^T S, upper tiles) with a single column of C beside it (ks_debug_time_gram, CUDA events)
  gram_gc  the G-Gram and the C-Gram (S^T R, k columns) in one launch, as ks_debug_time_gram issues them; gram_c = gram_gc - gram_g
  update   R += cbias - S W^T (gemm_kmajor_kernel, split update) through ks_debug_update, kernel time from torch.profiler (the debug
           entry splits its fp32 operands into fp16 pairs first; those kernels are not counted)
Executed TFLOP/s counts every launched 128 x 128 tile (three fp16 products each); smem_TBps counts the operand bytes the tiles
consume into shared memory (hi and lo planes of both operands: 1 KB per contraction row per tile, the same for every build).
"""
import argparse
import ctypes as C
import json
import sys

sys.path.insert(0, ".")
import keystone_b200 as ks  # noqa: E402
from keystone_b200._capi import KS_PRECISION_F16X2, check, lib  # noqa: E402

TILE = 128


def cdiv(a, b):
    return -(-a // b)


def g_tiles(b):
    nb = cdiv(b, TILE)
    return nb * (nb + 1) // 2


def rates(ms, tiles, contraction):
    flop = tiles * 3 * 2.0 * TILE * TILE * contraction
    smem = tiles * contraction * 4 * TILE * 2.0
    return {"ms": round(ms, 3), "tiles": tiles, "tflops": round(flop / ms / 1e9, 1), "smem_TBps": round(smem / ms / 1e9, 2)}


def time_gram(ctx, sa, sb, iters):
    ms = C.c_double(0)
    check(ctx.handle, lib().ks_debug_time_gram(ctx.handle, sa.handle, sb.handle, 2, C.byref(ms)))  # warm-up
    check(ctx.handle, lib().ks_debug_time_gram(ctx.handle, sa.handle, sb.handle, iters, C.byref(ms)))
    return ms.value


def time_update(ctx, sa, w, out, iters):
    import torch
    from torch.profiler import ProfilerActivity, profile

    def run():
        check(ctx.handle, lib().ks_debug_update(ctx.handle, sa.handle, w.handle, 0, KS_PRECISION_F16X2, None, 1, 2.0 ** -3,
                                                 out.handle))
    for _ in range(2):
        run()
    ctx.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            run()
        ctx.synchronize()
        torch.cuda.synchronize()
    times = [e.time_range.elapsed_us() for e in prof.events()
             if e.device_type == torch.autograd.DeviceType.CUDA and "gemm_kmajor_kernel" in e.name]
    if len(times) != iters:
        raise RuntimeError(f"expected {iters} update kernels in the trace, found {len(times)}")
    return sum(times) / iters / 1e3  # us -> ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 20)
    ap.add_argument("--block", type=int, default=4096)
    ap.add_argument("--classes", type=int, default=1000)
    ap.add_argument("--chunk-rows", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=5)
    a = ap.parse_args()
    n, b, k = a.rows, a.block, a.classes
    with ks.Context(0) as ctx:
        ctx.set_option("precision", 2)  # KS_PRECISION_F16X2: the debug entries split the operands and run the split kernels
        ctx.set_option("gram_chunk_rows", a.chunk_rows)
        sa = ctx.synthetic_normal(n, b, 11, 0)
        mb = cdiv(b, TILE)
        one = ctx.synthetic_normal(n, 1, 13, 0)
        t_g = time_gram(ctx, sa, one, a.iters)
        del one
        sb = ctx.synthetic_normal(n, k, 12, 0)
        t_gc = time_gram(ctx, sa, sb, a.iters)
        del sb
        common = {"rows": n, "block": b, "classes": k, "chunk_rows": a.chunk_rows}
        print(json.dumps({"kernel": "gram_g", **common, **rates(t_g, g_tiles(b) + mb, n)}), flush=True)
        print(json.dumps({"kernel": "gram_gc", **common, **rates(t_gc, g_tiles(b) + mb * cdiv(k, TILE), n)}), flush=True)
        print(json.dumps({"kernel": "gram_c", **common, **rates(t_gc - t_g, mb * (cdiv(k, TILE) - 1), n)}), flush=True)
        w = ctx.synthetic_normal(k, b, 14, 0)
        out = ctx.synthetic_normal(n, k, 15, 0)
        t_u = time_update(ctx, sa, w, out, a.iters)
        print(json.dumps({"kernel": "update", **common, **rates(t_u, cdiv(n, TILE) * cdiv(k, TILE), b)}), flush=True)


if __name__ == "__main__":
    main()
