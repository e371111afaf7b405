"""First-contact diagnostics for a GPU machine: prints rather than asserts, so one run
tells as much as possible.  Not part of the test-suite."""
import ctypes as C
import json
import os
import sys
import time
import traceback

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from layerskip_b200 import _lib
from layerskip_b200.engine import Engine
from layerskip_b200.weights import ARCHS, SyntheticLlama


def gemm_report():
    lib = _lib.load()
    for (n, k) in [(512, 256), (12288, 4096), (4096, 4096), (22016, 4096), (4096, 11008), (32000, 4096)]:
        for m in (1, 7, 16):
            if m > 8 and k > 8192:
                continue
            try:
                g = torch.Generator(device="cuda").manual_seed(1)
                w = (torch.randn(n, k, generator=g, device="cuda") * 0.02).to(torch.bfloat16)
                x = torch.randn(m, k, generator=g, device="cuda").to(torch.bfloat16)
                packed = torch.empty_like(w)
                _lib.check(lib.lsk_test_pack(w.data_ptr(), n, k, packed.data_ptr()))
                y = torch.zeros(m, n, dtype=torch.float32, device="cuda")
                ms = C.c_float(0)
                _lib.check(lib.lsk_test_gemm(packed.data_ptr(), n, k, x.data_ptr(), m, y.data_ptr(), 50, C.byref(ms)))
                ref = x.float() @ w.float().T
                err = float((y - ref).abs().max())
                gbs = n * k * 2 / (ms.value * 1e-3) / 1e9 if ms.value > 0 else 0
                print(f"gemm n={n:6d} k={k:6d} m={m:2d} max_err={err:.3e} ref_max={float(ref.abs().max()):.3f} "
                      f"avg_ms={ms.value:.4f} -> {gbs:8.1f} GB/s (L2-warm back-to-back)", flush=True)
            except Exception:
                traceback.print_exc()


def engine_report(arch_name, E, D, steps=64, prompt_len=32, alpha=1.0):
    arch = ARCHS[arch_name]
    t0 = time.time()
    model = SyntheticLlama(arch, seed=0, alpha=alpha, damp_from=E)
    eng = Engine(arch, max_ctx=2048)
    eng.load_model(model)
    torch.cuda.synchronize()
    print(f"[{arch_name}] engine ready in {time.time() - t0:.1f}s, params {arch.param_bytes() / 1e9:.2f} GB", flush=True)
    g = torch.Generator().manual_seed(1234)
    prompt = torch.randint(3, arch.vocab - 1, (prompt_len,), generator=g).tolist()
    for mode in ("spec", "ar"):
        eng.begin(exit_layer=E if mode == "spec" else -1, max_steps=steps, eos_token_ids=[arch.vocab - 1])
        t0 = time.time()
        eng.prefill(prompt)
        t_pre = time.time() - t0
        pre_ms = eng.last_device_ms
        out = []
        dev_ms = 0.0
        bytes_total = 0.0
        matches = drafted = 0
        n_rounds = 0
        t0 = time.time()
        while len(out) < steps:
            if mode == "spec":
                d = min(D, steps - len(out) - 1)
                ctx = eng.kv_len
                r = eng.round(d)
                out += r.emitted
                matches += r.n_matches
                drafted += r.n_drafted
                bytes_total += eng.round_bytes(d, ctx)
            else:
                ctx = eng.kv_len
                out.append(eng.ar_step())
                bytes_total += eng.ar_bytes(ctx)
            dev_ms += eng.last_device_ms
            n_rounds += 1
        wall = time.time() - t0
        print(f"[{arch_name}] {mode}: {len(out)} tok in {wall * 1e3:.1f} ms wall / {dev_ms:.1f} ms device "
              f"({len(out) / wall:.1f} tok/s), rounds={n_rounds}, acc={matches / max(1, drafted):.3f}, "
              f"prefill {t_pre * 1e3:.1f} ms (dev {pre_ms:.1f}), achieved {bytes_total / (dev_ms * 1e-3) / 1e9:.0f} GB/s, "
              f"launches={eng.launch_count}", flush=True)
        print("   first tokens:", out[:16], flush=True)
    eng.close()


if __name__ == "__main__":
    print(torch.cuda.get_device_name(0), torch.version.cuda, flush=True)
    what = sys.argv[1:] or ["gemm", "tiny", "small"]
    if "gemm" in what:
        gemm_report()
    try:
        if "tiny" in what:
            engine_report("tiny-gqa", 3, 6, steps=48, prompt_len=17, alpha=0.1)
        if "small" in what:
            engine_report("small-1b", 4, 6, steps=64, prompt_len=64, alpha=0.05)
        if "7b" in what:
            engine_report("llama2-7b", 8, 6, steps=128, prompt_len=128, alpha=1.0)
    except Exception:
        traceback.print_exc()
