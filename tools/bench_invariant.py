"""Cost of batch-invariant mode (ops.set_batch_invariant): the BASELINE config-2 workload of bench.py and the
tools/bench_serving.py request trace, each run with the mode off and on, alternated, in fresh processes.  Prints one
JSON line with the card name, power limit and SM clock beside the numbers.

The serving runs replay one arrival trace in both modes (--base-rate: every request arrives within microseconds), so
the engine's requests/s is its throughput on the same saturating workload, not a rate derived from each mode's own
single-request speed.

    python tools/bench_invariant.py [--rounds 2] [--steps 2 --warmup 1] [--requests 8 --serving-steps 20]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# runs `script` (a path under the repository) as __main__ with the given argv, in the requested mode
_RUNNER = """
import runpy, sys
sys.path[:0] = [{root!r}, {tools!r}]
from instancediffusion_b200 import ops
ops.set_batch_invariant({mode})
sys.argv = {argv!r}
runpy.run_path({script!r}, run_name="__main__")
"""


def _run(script, argv, mode):
    code = _RUNNER.format(root=ROOT, tools=os.path.join(ROOT, "tools"), mode=mode, argv=[script] + argv,
                          script=os.path.join(ROOT, script))
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, stdout=subprocess.PIPE, text=True, check=True)
    return json.loads([line for line in r.stdout.splitlines() if line.startswith("{")][-1])


def _gpu():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return dict(zip(q.split(","), [v.strip() for v in r.stdout.splitlines()[0].split(",")])) if r.returncode == 0 else {}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2, help="off / on pairs of each workload")
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--requests", type=int, default=8)
    ap.add_argument("--serving-steps", type=int, default=20)
    args = ap.parse_args()
    out = {"gpu": _gpu(), "config2_images_per_s": {"off": [], "on": []}, "engine_requests_per_s": {"off": [], "on": []}}
    for _ in range(args.rounds):
        for mode in (False, True):
            key = "on" if mode else "off"
            b = _run("bench.py", ["--gpus", "1", "--steps", str(args.steps), "--warmup", str(args.warmup),
                                  "--no-cpu-baseline", "--no-mis-leg"], mode)
            out["config2_images_per_s"][key].append(b.get("value", b))
            s = _run("tools/bench_serving.py", ["--requests", str(args.requests), "--steps", str(args.serving_steps),
                                                "--load", "1.0", "--base-rate", "1000"], mode)
            load = s["loads"]["1.0"]
            out["engine_requests_per_s"][key].append(load["engine"]["requests_per_s"])
            out.setdefault("engine_clocks", {}).setdefault(key, []).append(load["engine"]["clocks"])
            print(f"[bench_invariant] mode {key}: config 2 {out['config2_images_per_s'][key][-1]:.3f} images/s, engine "
                  f"{out['engine_requests_per_s'][key][-1]:.3f} requests/s", file=sys.stderr, flush=True)
    for k in ("config2_images_per_s", "engine_requests_per_s"):
        v = out[k]
        v["mean"] = {m: sum(v[m]) / len(v[m]) for m in ("off", "on")}
        v["on_vs_off"] = v["mean"]["on"] / v["mean"]["off"] - 1
    out["gpu_after"] = _gpu()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
