#!/usr/bin/env python
"""GEMM shapes of the APE-L_D step with the epilogues the model uses, timed as CUDA-graph replays (no host launch cost in
the number) and dissected by the kernel's own clock64 stamps (ape_gemm_set_trace).  Development aid.

    python tests/perf_gemm2.py > gpurun_out/gemm_phases.jsonl

Per shape and variant: us per launch (graph of 20 launches, warm operands; `cold` = 8 rotating weight / activation sets larger
than L2 together), TFLOP/s, and medians over CTAs of the phases in SM cycles:
  setup   entry -> barriers ready                        load   -> first operands landed
  issue   first operands -> last MMA issued           acc1   first operands -> first accumulator complete
  tail    last accumulator complete -> stores drained total  entry -> exit"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ape_b200  # noqa: E402,F401
from ape_b200 import _lib, ops  # noqa: E402

DEV = "cuda:0"
SHAPES = [  # (what, M, N, K, act, epilogue, count per step)
    ("vit qkv", 4096, 3072, 1024, None, "f16", 24),
    ("vit proj", 4096, 1024, 1024, None, "f32+res+ln", 24),
    ("vit w12", 4096, 5460, 1024, "swiglu", "f16+stats", 24),
    ("vit w3", 4096, 1024, 2730, None, "f32+res+ln", 24),
    ("enc ffn1", 87296, 2048, 256, "relu", "f16", 6),
    ("enc ffn2", 87296, 256, 2048, None, "f32+res", 6),
    ("enc 256x256", 87296, 256, 256, None, "f16", 21),
    ("enc qo", 87296, 480, 256, None, "f16", 6),
    ("dec 256x256", 900, 256, 256, None, "f16", 31),
    ("dec ffn1", 900, 2048, 256, "relu", "f16", 6),
    ("dec ffn2", 900, 256, 2048, None, "f32+res", 6),
]
VARIANTS = {"single": 0x1000, "mc2": 0x4000}
if os.environ.get("PERF_GEMM_VARIANTS"):
    VARIANTS = {k: v for k, v in VARIANTS.items() if k in os.environ["PERF_GEMM_VARIANTS"].split(",")}


def make_case(M, N, K, act, epi, nsets):
    Kp = (K + 7) // 8 * 8
    n_out = N // 2 if act == "swiglu" else N
    sets = []
    for _ in range(nsets):
        x = torch.randn(M, Kp, device=DEV, dtype=torch.float16)[:, :K]
        w = (torch.randn(N, Kp, device=DEV, dtype=torch.float16) * K ** -0.5)[:, :K]
        b = torch.randn(N, device=DEV)
        kw = {}
        if epi.startswith("f32"):
            out = torch.empty(M, n_out, device=DEV, dtype=torch.float32)
            if "res" in epi:
                kw["residual"] = torch.randn(M, n_out, device=DEV, dtype=torch.float32)
            if "ln" in epi:
                nparts = (K + 63) // 64
                part = torch.zeros(M, nparts, 2, device=DEV)
                xf = x.float()
                for i in range(nparts):
                    sl = xf[:, 64 * i:64 * i + 64]
                    part[:, i, 0], part[:, i, 1] = sl.sum(1), (sl * sl).sum(1)
                kw["ln_fold"] = (part, w.float().sum(1).contiguous(), K, 1e-6)
        else:
            out = torch.empty(M, (n_out + 7) // 8 * 8, device=DEV, dtype=torch.float16)[:, :n_out]
            if "stats" in epi:
                kw["stats_out"] = True
        sets.append((x, w, b, out, kw))
    return sets


def run(sets, act, tile, i):
    x, w, b, out, kw = sets[i % len(sets)]
    return ops.linear_tc(x, w, b, act=act, tile_n=256 | tile if w.shape[0] > 128 else tile, out=out, **kw)


class Clocks:
    """SM clock / power sampled by NVML in a thread while a measurement runs."""

    def __init__(self):
        import threading

        import pynvml
        pynvml.nvmlInit()
        self.nv, self.h = pynvml, pynvml.nvmlDeviceGetHandleByIndex(0)
        self.samples, self.stop = [], threading.Event()
        self.t = threading.Thread(target=self._loop, daemon=True)

    def _loop(self):
        while not self.stop.is_set():
            try:
                self.samples.append((self.nv.nvmlDeviceGetClockInfo(self.h, self.nv.NVML_CLOCK_SM), self.nv.nvmlDeviceGetPowerUsage(self.h) / 1e3))
            except Exception:  # noqa: BLE001
                pass
            self.stop.wait(0.02)

    def __enter__(self):
        self.t.start()
        return self

    def __exit__(self, *exc):
        self.stop.set()
        self.t.join()
        return False

    def summary(self):
        if not self.samples:
            return None
        c = sorted(x[0] for x in self.samples)
        return {"sm_mhz_median": c[len(c) // 2], "sm_mhz_min": c[0], "power_w_max": round(max(x[1] for x in self.samples)), "n": len(c)}


def graph_time(sets, act, tile, launches=20, reps=10):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for i in range(len(sets)):
            run(sets, act, tile, i)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(launches):
            run(sets, act, tile, i)
    g.replay()
    torch.cuda.synchronize()
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        g.replay()
    e.record()
    torch.cuda.synchronize()
    return a.elapsed_time(e) / (reps * launches) * 1e3


def sustained(sets, act, tile, seconds=1.5):
    """The same graph replayed back to back for `seconds`: (us per launch, clocks under that load)."""
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(20):
            run(sets, act, tile, i)
    g.replay()
    torch.cuda.synchronize()
    import time
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 0
    with Clocks() as ck:
        t0 = time.time()
        a.record()
        while time.time() - t0 < seconds:
            for _ in range(20):
                g.replay()
            n += 20
            torch.cuda.synchronize()
        e.record()
        torch.cuda.synchronize()
    return a.elapsed_time(e) / (n * 20) * 1e3, ck.summary()


def phases(sets, act, tile):
    buf = torch.zeros(torch.cuda.get_device_properties(DEV).multi_processor_count * 8 * 2, dtype=torch.int64, device=DEV)
    _lib.lib.ape_gemm_set_trace(buf.data_ptr())
    try:
        run(sets, act, tile, 0)
        torch.cuda.synchronize()
    finally:
        _lib.lib.ape_gemm_set_trace(None)
    t = buf.view(-1, 8).cpu()
    t = t[t[:, 0] != 0]
    if t.numel() == 0:
        return None
    t = t.double()
    med = lambda v: int(v.median().item())  # noqa: E731
    return {"ctas": int(t.shape[0]), "setup": med(t[:, 1] - t[:, 0]), "load": med(t[:, 2] - t[:, 1]), "issue": med(t[:, 3] - t[:, 2]),
            "acc1": med(t[:, 4] - t[:, 2]), "acc_last_from_entry": med(t[:, 5] - t[:, 0]), "tail": med(t[:, 6] - t[:, 5]),
            "total": med(t[:, 7] - t[:, 0]), "total_max": int((t[:, 7] - t[:, 0]).max().item())}


def main():
    os.environ.setdefault("APE_PDL", "0")  # back-to-back launches of one kernel: no overlap, clean per-launch numbers
    for (what, M, N, K, act, epi, cnt) in SHAPES:
        flops = 2.0 * M * N * K
        warm = make_case(M, N, K, act, epi, 1)
        per_set = M * K * 2 + N * K * 2 + M * (N // 2 if act == "swiglu" else N) * (4 if epi.startswith("f32") else 2)
        cold = make_case(M, N, K, act, epi, max(2, min(8, int(300e6 // per_set) + 1)))
        for name, tile in VARIANTS.items():
            rec = {"what": what, "M": M, "N": N, "K": K, "epilogue": epi, "variant": name, "per_step": cnt}
            try:
                us = graph_time(warm, act, tile)
                rec.update(us_warm=round(us, 2), tflops_warm=round(flops / us / 1e6, 1))
                us = graph_time(cold, act, tile)
                rec.update(us_cold=round(us, 2), tflops_cold=round(flops / us / 1e6, 1), cold_sets=len(cold),
                           ms_per_step_cold=round(us * cnt / 1e3, 3))
                rec["cycles"] = phases(warm, act, tile)
                if name == "single" and M >= 4096:
                    us, ck = sustained(warm, act, tile)
                    rec.update(us_sustained=round(us, 2), tflops_sustained=round(flops / us / 1e6, 1), clocks_sustained=ck)
            except Exception as ex:  # noqa: BLE001
                rec["error"] = str(ex)[:300]
            print(json.dumps(rec), flush=True)
        del warm, cold
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
