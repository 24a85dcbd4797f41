"""GPU bring-up of the wgmma GEMM core: every variant in its own subprocess (a trapped kernel
poisons the CUDA context), results appended to gpurun_out/bringup_gemm.jsonl."""
import ctypes as C
import json
import os
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
OUT = ROOT / "gpurun_out"


def child(variant: int, fmt: int, M: int, N: int, K: int, epi: int):
    import torch
    lib = C.CDLL(str(ROOT / "ance_b200" / "lib" / "libance_b200.so"))
    lib.ance_dbg_gemm.restype = C.c_int
    lib.ance_dbg_gemm.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                  C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.ance_last_error.restype = C.c_char_p
    torch.manual_seed(0)
    dt = torch.bfloat16 if fmt == 1 else torch.float16
    dev = "cuda:0"
    A = (torch.randn(M, K, device=dev) * 0.5).to(dt)
    B = (torch.randn(N, K, device=dev) * 0.5).to(dt)
    bias = torch.randn(N, device=dev) if epi else None
    R = torch.randn(M, N, device=dev).to(torch.bfloat16) if epi else None
    C32 = torch.full((M, N), float("nan"), device=dev)
    C16 = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
    st = torch.cuda.current_stream().cuda_stream
    rc = lib.ance_dbg_gemm(A.data_ptr(), B.data_ptr(), M, N, K, fmt, variant,
                           bias.data_ptr() if epi else None, R.data_ptr() if epi else None, 1 if epi else 0,
                           C16.data_ptr(), C32.data_ptr(), st)
    if rc != 0:
        print(json.dumps({"ok": False, "err": lib.ance_last_error().decode()}))
        return
    torch.cuda.synchronize()
    ref = A.float() @ B.float().t()
    if epi:
        ref = torch.nn.functional.gelu(ref + bias) + R.float()
    err = (C32 - ref).abs().max().item()
    err16 = (C16.float() - ref).abs().max().item()
    if epi:  # bf16-only output with residual: the TMA-residual path of the epilogue
        C16b = torch.zeros_like(C16)
        lib.ance_dbg_gemm(A.data_ptr(), B.data_ptr(), M, N, K, fmt, variant, bias.data_ptr(), R.data_ptr(), 1,
                          C16b.data_ptr(), None, st)
        torch.cuda.synchronize()
        err16 = max(err16, (C16b.float() - ref).abs().max().item())
    nan = int(torch.isnan(C32).sum().item())
    # timing
    for _ in range(3):
        lib.ance_dbg_gemm(A.data_ptr(), B.data_ptr(), M, N, K, fmt, variant, None, None, 0, C16.data_ptr(), None, st)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    iters = 10
    for _ in range(iters):
        lib.ance_dbg_gemm(A.data_ptr(), B.data_ptr(), M, N, K, fmt, variant, None, None, 0, C16.data_ptr(), None, st)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    tf = 2.0 * M * N * K / ms / 1e9
    print(json.dumps({"ok": bool(err < 0.05 and err16 < 0.3 and nan == 0), "max_err_f32": err, "max_err_bf16": err16, "nan": nan,
                      "ms": ms, "tflops": tf}))


def main():
    OUT.mkdir(exist_ok=True)
    cases = []
    # (variant, fmt, M, N, K, epi)
    for v in (0, 1, 4, 2, 3):
        cases.append((v, 1, 256, 512, 128, 0))       # tiny: descriptor sanity
        cases.append((v, 1, 1000, 776, 768, 1))      # ragged M/N + epilogue
        cases.append((v, 1, 8192, 3072, 768, 0))     # encoder FFN-up shape
        cases.append((v, 0, 8192, 768, 3072, 0))     # fp16, FFN-down shape
    cases.append((0, 1, 65536, 2304, 768, 0))
    cases.append((2, 1, 65536, 2304, 768, 0))
    with open(OUT / "bringup_gemm.jsonl", "a") as f:
        for c in cases:
            t0 = time.time()
            try:
                r = subprocess.run([sys.executable, __file__, "child", *map(str, c)], capture_output=True, text=True,
                                   timeout=120)
                line = (r.stdout.strip().splitlines() or ["{}"])[-1]
                try:
                    res = json.loads(line)
                except Exception:
                    res = {"ok": False, "stdout": r.stdout[-2000:]}
                res["rc"] = r.returncode
                if r.returncode != 0:
                    res["stderr"] = r.stderr[-1500:]
                    res["stdout"] = r.stdout[-1500:]
            except subprocess.TimeoutExpired:
                res = {"ok": False, "timeout": True}
            res["case"] = c
            res["wall_s"] = round(time.time() - t0, 1)
            print(json.dumps(res), flush=True)
            f.write(json.dumps(res) + "\n")
            f.flush()


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "child":
        child(*map(int, sys.argv[2:]))
    else:
        main()
