"""Bring-up check for cv_gemm_bf16 on a real H100: every operand-major combination, tile width and
epilogue, each case in its own subprocess (a trap poisons the CUDA context) under a timeout.

    python tools/gemm_check.py            # run all cases, write gpurun_out/gemm_check.json
    python tools/gemm_check.py --case N   # run one case in-process
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = [
    # name, M, N, K, a_mn, b_mn, block_n, out_f32, bias, act, absmax, preact
    ("tn_128", 256, 256, 256, 0, 0, 128, 0, 0, 0, 0, 0),
    ("tn_256", 256, 512, 256, 0, 0, 256, 0, 0, 0, 0, 0),
    ("tn_128_k64", 128, 128, 64, 0, 0, 128, 0, 0, 0, 0, 0),
    ("tn_big", 4352, 7680, 2560, 0, 0, 0, 0, 1, 0, 0, 0),
    ("tn_f32", 256, 384, 512, 0, 0, 128, 1, 1, 0, 1, 0),
    ("tn_gelu", 384, 1024, 256, 0, 0, 256, 0, 1, 1, 1, 1),
    ("tn_ragged", 200, 328, 136, 0, 0, 0, 0, 1, 0, 1, 0),
    ("dgrad_128", 256, 256, 384, 0, 1, 128, 0, 0, 0, 0, 0),
    ("dgrad_256", 384, 512, 256, 0, 1, 256, 0, 0, 0, 0, 0),
    ("wgrad_128", 256, 384, 512, 1, 1, 128, 0, 0, 0, 0, 0),
    ("wgrad_256", 512, 256, 1088, 1, 1, 256, 0, 0, 0, 0, 0),
    ("wgrad_ragged", 200, 328, 1000, 1, 1, 0, 0, 0, 0, 0, 0),
    ("logits", 264, 58240, 256, 0, 0, 0, 1, 0, 0, 0, 0),
]


def run_case(i):
    import torch
    from cogview_b200 import ops
    name, M, N, K, a_mn, b_mn, bn, out_f32, use_bias, act, use_absmax, preact = CASES[i]
    g = torch.Generator(device="cuda").manual_seed(i)
    A = torch.randn((K, M) if a_mn else (M, K), device="cuda", generator=g).to(torch.bfloat16)
    B = torch.randn((K, N) if b_mn else (N, K), device="cuda", generator=g).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g).to(torch.bfloat16) if use_bias else None
    absmax = torch.zeros(1, device="cuda", dtype=torch.float32) if use_absmax else None
    res = ops.gemm(A, B, a_mn_major=bool(a_mn), b_mn_major=bool(b_mn), bias=bias, act=act,
                   out_dtype=torch.float32 if out_f32 else torch.bfloat16, absmax=absmax,
                   want_preact=bool(preact), block_n=bn)
    torch.cuda.synchronize()
    C, pre = (res if preact else (res, None))
    Af = (A.t() if a_mn else A).float()
    Bf = (B.t() if b_mn else B).float()
    ref = Af @ Bf.t()
    if use_bias:
        ref = ref + bias.float()
    ref_pre = ref
    if act:
        ref = 0.5 * ref * (1.0 + torch.tanh(0.7978845608028654 * ref * (1.0 + 0.044715 * ref * ref)))
    err = (C.float() - ref).abs().max().item()
    scale = ref.abs().max().item()
    out = {"name": name, "max_abs_err": err, "ref_scale": scale, "rel": err / max(scale, 1e-9)}
    if preact:
        out["preact_err"] = (pre.float() - ref_pre).abs().max().item()
    if use_absmax:
        tgt = (C.float().abs().max().item())
        out["absmax"] = absmax.item()
        out["absmax_expected"] = tgt
    tol = 2e-2 if not out_f32 else 2e-3
    out["ok"] = bool(out["rel"] < tol and (not use_absmax or abs(out["absmax"] - out["absmax_expected"]) <= 1e-6 * max(1, tgt)))
    # timing for the big case
    if M * N * K > 1e10:
        for _ in range(3):
            ops.gemm(A, B, a_mn_major=bool(a_mn), b_mn_major=bool(b_mn), bias=bias, act=act, block_n=bn)
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        iters = 20
        for _ in range(iters):
            ops.gemm(A, B, a_mn_major=bool(a_mn), b_mn_major=bool(b_mn), bias=bias, act=act, block_n=bn)
        e.record()
        torch.cuda.synchronize()
        ms = s.elapsed_time(e) / iters
        out["ms"] = ms
        out["tflops"] = 2.0 * M * N * K / ms / 1e9
        s.record()
        for _ in range(iters):
            torch.matmul((A.t() if a_mn else A), (B if b_mn else B.t()))
        e.record()
        torch.cuda.synchronize()
        out["cublas_tflops"] = 2.0 * M * N * K / (s.elapsed_time(e) / iters) / 1e9
    print("RESULT " + json.dumps(out))


def main():
    if "--case" in sys.argv:
        run_case(int(sys.argv[sys.argv.index("--case") + 1]))
        return
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    results = []
    for i, c in enumerate(CASES):
        try:
            r = subprocess.run([sys.executable, __file__, "--case", str(i)], capture_output=True, text=True,
                               timeout=180)
            line = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")]
            if line:
                results.append(json.loads(line[0][7:]))
            else:
                results.append({"name": c[0], "ok": False, "rc": r.returncode, "stderr": r.stderr[-600:]})
        except subprocess.TimeoutExpired:
            results.append({"name": c[0], "ok": False, "error": "timeout"})
        print(json.dumps(results[-1]), flush=True)
    with open(os.path.join(ROOT, "gpurun_out", "gemm_check.json"), "w") as f:
        json.dump(results, f, indent=1)
    print("PASSED %d / %d" % (sum(1 for r in results if r.get("ok")), len(results)))


if __name__ == "__main__":
    main()
