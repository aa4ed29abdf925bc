"""HBM-cold timings (weights rotating over the 32 layers, CUDA-graph replay) of the decoder's latency-bound pieces at the benchmarked
shape: the swap-AB GEMMs one launch at a time, the split-K reduce, self-attention and cross-attention.

    python tools/microbench_cold.py [batch]
"""
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

if __name__ == "__main__":
    import whisperkit_b200 as wk
    from whisperkit_b200._lib import check
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 64
    m = wk.Model("large-v3", max_batch=B)
    m.init_random(1)
    dec = wk.TextDecoder(m, B)
    names = {14: "d x d GEMM (out / cross-Q / cross-out)", 17: "QKV GEMM", 15: "FC1 GEMM", 16: "FC2 GEMM", 8: "split-K reduce + LN",
             9: "self-attention @ pos 100", 0: "cross-attention"}
    f, w = C.c_float(), C.c_double()
    for k, n in names.items():
        check(m.lib.wk_bench_kernel(m.handle, dec.handle, k, B, 192, C.byref(f), C.byref(w)))
        gbs = w.value / (f.value * 1e-3) / 1e9 if w.value else 0.0
        print(f"{n:58s} {f.value * 1000:8.2f} us   {gbs:8.0f} GB/s of algorithmic bytes", flush=True)
