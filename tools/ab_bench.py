"""A/B of two builds of the library on bench.py: N runs of each, alternated, one subprocess at a time.
Usage: python tools/ab_bench.py LIB_A LIB_B [runs per library = 5] [extra bench.py arguments, e.g. --config 2]
LIB_A / LIB_B: paths of two libptts_b200*.so (csrc/build.py --tag NAME), loaded through PTTS_LIB; `product` = the product library.
Prints the median and the spread (max - min over the median) of `value`, `e2e.value` and `roofline.ms_per_decode_step` per
library, B against A, whether every run of B beat every run of A, and the card the numbers belong to."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = {"value": lambda d: d["value"], "e2e.value": lambda d: d["e2e"]["value"], "roofline.ms_per_decode_step": lambda d: d["roofline"]["ms_per_decode_step"]}


def run(lib, extra):
    env = dict(os.environ)
    env.pop("PTTS_LIB", None)
    if lib != "product":
        env["PTTS_LIB"] = os.path.abspath(lib)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--no-cpu-baseline", "--no-gpu-reference", *extra],
                       env=env, cwd=ROOT, capture_output=True, text=True)
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    if r.returncode != 0 or not lines:
        raise RuntimeError(f"bench.py failed with {lib} (exit {r.returncode}):\n{r.stdout[-2000:]}\n{r.stderr[-2000:]}")
    return json.loads(lines[-1])


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:
        return f"nvidia-smi unavailable ({ex!r})"


def main():
    libs = sys.argv[1:3]
    rest = sys.argv[3:]
    n = int(rest.pop(0)) if rest and rest[0].isdigit() else 5
    res = {lib: [] for lib in libs}
    for i in range(n):
        for lib in libs:
            d = run(lib, rest)
            res[lib].append(d)
            print(f"run {i} {lib}: " + "  ".join(f"{k} {f(d):.6g}" for k, f in KEYS.items()) + f"  clocks {d.get('clocks')}", flush=True)
    print(f"\ncard (name, power limit, max SM clock): {card()}")
    for k, f in KEYS.items():
        v = {lib: np.array([f(d) for d in res[lib]]) for lib in libs}
        med = {lib: float(np.median(v[lib])) for lib in libs}
        a, b = libs
        better = (v[b].max() < v[a].min()) if k.endswith("step") else (v[b].min() > v[a].max())
        print(f"{k}: " + "  ".join(f"{lib} median {med[lib]:.6g} spread {100 * (v[lib].max() - v[lib].min()) / med[lib]:.2f} %" for lib in libs)
              + f"  B/A {100 * (med[b] / med[a] - 1):+.2f} %  every B run better than every A run: {bool(better)}")
    os.makedirs(os.path.join(ROOT, "tools_out"), exist_ok=True)
    json.dump({"card": card(), "args": rest, "runs": res}, open(os.path.join(ROOT, "tools_out", "ab_bench.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
