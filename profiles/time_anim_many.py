"""One update_many over a frame's animation systems against the loop of per-system updates it replaces (DESIGN.md §4.3).

  0. probe: launch cost of an empty kernel by the size of its __grid_constant__ parameter block (256 B .. 32000 B), host enqueue and
     device time per launch over back-to-back launches (a tiny CUDA program built with nvcc into a temporary directory)
  1. config 4 as one system (100 k instances x 64 bones, DQ palette): update_many([s]) against update(s)
  2. 100 k instances over 32 systems of 16-196 bones: one update_many against 32 updates
  3. 256 systems x 64 instances (the launch-bound case): the same two forms
  4. one 196-bone system + 63 systems of 20 bones: the batched call against the 20-bone systems batched alone plus the 196-bone one alone
     (the residency cost of sizing shared memory for the largest skeleton)
Device time: CUDA events around `calls` calls; host time: first enqueue to the end of a synchronise.  Forms alternate window by window,
every shape is warmed up first, and the medians and spreads of the windows are printed with the card, its power limit and its maximum
SM clock, read in the same run.  Both forms are checked to leave byte-equal outputs before anything is timed.
Usage: python profiles/time_anim_many.py [windows] [calls_per_window]"""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lumixengine_b200 as lb  # noqa: E402
from lumixengine_b200 import scenes  # noqa: E402

PROBE = r"""
#include <cstdio>
#include <chrono>
#include <cuda_runtime.h>
template <int BYTES> struct P { unsigned w[BYTES / 4]; };
template <int BYTES> __global__ void k(const __grid_constant__ P<BYTES> p) { if (p.w[threadIdx.x % (BYTES / 4)] == 0xdeadbeef) printf("x"); }
template <int BYTES> void run(cudaStream_t s, int n) {
	P<BYTES> p = {};
	for (int i = 0; i < 200; ++i) k<BYTES><<<1, 32, 0, s>>>(p);
	cudaStreamSynchronize(s);
	cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
	auto t0 = std::chrono::steady_clock::now();
	cudaEventRecord(a, s);
	for (int i = 0; i < n; ++i) k<BYTES><<<1, 32, 0, s>>>(p);
	cudaEventRecord(b, s);
	auto t1 = std::chrono::steady_clock::now();
	cudaEventSynchronize(b);
	float ms = 0; cudaEventElapsedTime(&ms, a, b);
	printf("{\"param_bytes\": %d, \"host_enqueue_us\": %.3f, \"device_us\": %.3f}\n", BYTES,
		std::chrono::duration<double, std::micro>(t1 - t0).count() / n, 1000.0 * ms / n);
}
int main() {
	cudaStream_t s; cudaStreamCreate(&s);
	for (int r = 0; r < 3; ++r) { run<256>(s, 5000); run<4096>(s, 5000); run<10512>(s, 5000); run<21008>(s, 5000); run<32000>(s, 5000); }
	return cudaGetLastError() != cudaSuccess;
}
"""


def probe():
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "probe.cu"), os.path.join(d, "probe")
        open(src, "w").write(PROBE)
        subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe, src])
        rows = [json.loads(line) for line in subprocess.check_output([exe], text=True).splitlines() if line.startswith("{")]
    out = {}
    for r in rows:
        out.setdefault(r["param_bytes"], []).append((r["host_enqueue_us"], r["device_us"]))
    return {b: {"host_enqueue_us": float(np.median([x[0] for x in v])), "device_us": float(np.median([x[1] for x in v]))} for b, v in out.items()}


def card():
    q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True)
    return q.strip().splitlines()[0]


def systems(ctx, specs, seed, palette):
    """Two identical lists of systems (one per form) for specs = [(bones, instances)]."""
    out = ([], [])
    for k, (bones, n) in enumerate(specs):
        sk = scenes.skeleton(bones, seed=bones)
        clips = [scenes.clip(sk, frames=30, seed=seed + k), scenes.clip(sk, frames=45, seed=seed + k + 1000)]
        ci, tt = scenes.instance_times(n, clips, seed=seed + k)
        for side in out:
            s = lb.AnimationSystem(ctx, sk, clips, None, max_instances=n)
            s.setInstances(ci, tt)
            side.append(s)
    many, one = out
    lb.AnimationSystem.updateMany(many, 1.0 / 60.0, palette)
    for s in one:
        s.update(1.0 / 60.0, palette)
    for a, b in zip(many, one):
        assert a.getDualQuats().tobytes() == b.getDualQuats().tobytes() and a.getTimes().tobytes() == b.getTimes().tobytes()
    return many, one


def timed(ctx, forms, windows, calls):
    """forms: name -> callable of one frame.  Alternating windows; per form the medians (and min..max) of device and host ms per call."""
    e0, e1 = ctx.event(), ctx.event()
    res = {k: {"device": [], "host": []} for k in forms}
    for f in forms.values():  # warm-up of every shape
        for _ in range(3):
            f()
    ctx.synchronize()
    for w in range(windows):
        for name, f in (forms.items() if w % 2 == 0 else reversed(list(forms.items()))):
            ctx.synchronize()
            t0 = time.perf_counter()
            ctx.record(e0)
            for _ in range(calls):
                f()
            ctx.record(e1)
            ctx.synchronize()
            res[name]["host"].append((time.perf_counter() - t0) * 1e3 / calls)
            res[name]["device"].append(ctx.elapsed_ms(e0, e1) / calls)
    return {k: {m: {"median_ms": float(np.median(v[m])), "min_ms": float(np.min(v[m])), "max_ms": float(np.max(v[m]))} for m in v} for k, v in res.items()}


def main():
    windows = int(sys.argv[1]) if len(sys.argv) > 1 else 9
    calls = int(sys.argv[2]) if len(sys.argv) > 2 else 20
    ctx = lb.Context(0)
    out = {"card": card(), "probe": probe()}
    DQ = lb.PALETTE_DUAL_QUAT
    dt = 1.0 / 60.0
    rng = np.random.default_rng(1)
    cases = {
        "1_c4_one_system": [(64, 100_000)],
        "2_100k_over_32_systems": [(int(b), 100_000 // 32) for b in rng.integers(16, 197, 32)],
        "3_256_systems_x_64": [(int(b), 64) for b in rng.integers(16, 197, 256)],
    }
    for name, specs in cases.items():
        many, one = systems(ctx, specs, 10, DQ)
        out[name] = timed(ctx, {"update_many": lambda: lb.AnimationSystem.updateMany(many, dt, DQ),
                                "update_loop": lambda: [s.update(dt, DQ) for s in one]}, windows, calls)
        for s in many + one:
            s.close()
    # 4: residency — 63 x 20-bone systems of 1600 instances with and without one 196-bone system of 1600 instances in the same launch
    small, _ = systems(ctx, [(20, 1600)] * 63, 20, DQ)
    big, _ = systems(ctx, [(196, 1600)], 30, DQ)
    out["4_196_with_63_x_20"] = timed(ctx, {"mixed": lambda: lb.AnimationSystem.updateMany(big + small, dt, DQ),
                                            "small_alone": lambda: lb.AnimationSystem.updateMany(small, dt, DQ),
                                            "big_alone": lambda: lb.AnimationSystem.updateMany(big, dt, DQ)}, windows, calls)
    print(json.dumps(out, indent=1))
    ctx.close()


if __name__ == "__main__":
    main()
