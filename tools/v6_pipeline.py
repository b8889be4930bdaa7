"""Where the exact sampler's draw period goes: cycles per draw of each pipeline role of
`exact_deep_v6` (pfrl_b200/csrc/tree_dev.cuh) on bench.py's headline pass.

Builds libb2rl.so with -DB2RL_V6_PROFILE=1 (clock64 sums per pipeline segment) into OUT,
leaving the in-tree library alone, runs bench.py's exact-sampler pass on it with
B2RL_V6_CYCLES=1 (1 M-leaf tree, B = 512, one k_replay_step launch per pass) and prints,
with the card name and power limit:

  main    own work: decide + table loads + stores; waits: for its scout (the next draw's
          staging), and the segment that held the ascent-queue check (now the root update only);
          the scout wait split into draws whose staging was not yet released when it was
          prefetched (spin and reload, and how many such draws) and the issue of the next
          draw's prefetch, which waits for its ready word
  ascent  work and wait per draw, summed over the V6_NASC ascent warps; the warps apply
          draws side by side, so the draw period they set is work / V6_NASC
  scouts  fast / slow draws of the last pass

The counters of the LAST launch are read; the profiled build is slower than the plain one,
so its samples/s are not the headline number.

    python tools/v6_pipeline.py --out /tmp/v6prof [--steps 4 --warmup 2]
"""
import argparse
import contextlib
import io
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def nasc():
    src = open(os.path.join(ROOT, "pfrl_b200", "csrc", "tree_dev.cuh")).read()
    return int(re.search(r"constexpr int V6_NASC = (\d+);", src).group(1))


def build_profiled(out):
    from pfrl_b200 import _lib

    lib = os.path.join(out, "libb2rl_v6profile.so")
    nvcc = os.environ.get("NVCC", "nvcc")
    subprocess.check_call([nvcc] + _lib.NVCC_FLAGS + ["-DB2RL_V6_PROFILE=1", "-I", _lib.INCLUDE,
                                                      "-o", lib] + _lib._sources())
    return lib


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for the profiled library and results")
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    lib = build_profiled(args.out)

    os.environ["B2RL_V6_CYCLES"] = "1"  # read once by the library, before the first launch
    from pfrl_b200 import _lib

    _lib.LIB_PATH = lib
    # bench.py reports a fixed subset of b2rl_step_times; keep the whole array of the last call
    L = _lib.load()
    step_times = L.b2rl_step_times
    raw = []

    def keep_step_times(h, ph, stream):
        st = step_times(h, ph, stream)
        raw[:] = list(ph)
        return st

    L.b2rl_step_times = keep_step_times
    import bench

    sys.argv = ["bench.py", "--no-rainbow", "--no-secondary", "--no-cpu-baseline",
                "--steps", str(args.steps), "--warmup", str(args.warmup)]
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        bench.main()
    line = json.loads(buf.getvalue().strip().splitlines()[-1])
    with open(os.path.join(args.out, "bench_profiled.json"), "w") as f:
        json.dump(line, f)

    ph = line["roofline"]["phases_of_one_launch"]
    c = ph["sampler_cycles_per_draw"]
    s = line["sampler"]
    na = nasc()
    main_work = c["main_decide"] + c["main_loads"] + c["main_stores"]
    B = line["config"]["batch_per_rank"]
    late, n_late, pref = raw[9] / B, raw[10], raw[11] / B  # dbg_cycles [5], [6], [7]
    res = {
        "card": card(),
        "ascent_warps": na,
        "main": {"own_work": main_work, "decide": c["main_decide"], "loads": c["main_loads"],
                 "stores": c["main_stores"], "wait_scout": c["main_wait_scout"],
                 "late_scout": late, "late_draws": n_late, "prefetch_next": pref,
                 "wait_queue": c["main_wait_queue"]},
        "ascent": {"work_per_draw": c["ascent_work"], "wait_per_draw": c["ascent_wait"],
                   "work_per_draw_period": c["ascent_work"] / na},
        "draw_period_cycles": main_work + c["main_wait_scout"] + c["main_wait_queue"],
        "sampling_us": ph["sampling_us"],
        "fast_draws": s["fast_draws"], "slow_draws": s["slow_draws"],
        "samples_per_sec_profiled_build": line["value"],
    }
    with open(os.path.join(args.out, "v6_pipeline.json"), "w") as f:
        json.dump(res, f, indent=1)
    print("card: %s" % res["card"])
    print("cycles per draw (last launch, B = %d):" % B)
    print("  main    own work %6.0f  (decide %.0f, table loads %.0f, stores %.0f)"
          % (main_work, c["main_decide"], c["main_loads"], c["main_stores"]))
    print("          waits    for its scout %.0f, queue segment %.0f"
          % (c["main_wait_scout"], c["main_wait_queue"]))
    print("          scout not released at the prefetch: %.0f (%d of %d draws); issuing the next"
          " draw's prefetch: %.0f" % (late, n_late, B, pref))
    print("  ascent  work %6.0f per draw over %d warps = %.0f per draw period; wait %.0f"
          % (c["ascent_work"], na, c["ascent_work"] / na, c["ascent_wait"]))
    print("  draw period (main work + waits) %.0f; sampling phase %.1f us"
          % (res["draw_period_cycles"], ph["sampling_us"]))
    print("  draws: %d fast, %d slow" % (s["fast_draws"], s["slow_draws"]))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
