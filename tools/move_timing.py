"""Device time of one map move (ElevationMap.move_to with a non-zero cell shift: k_shift into the shift buffer and the
copy back into the state buffer) at 1024^2 and 2048^2 (DESIGN.md §4b).

The handle runs on a torch stream; CUDA events on that stream bracket --moves calls of move_to that alternate between
two positions 3 and 2 cells apart, after a warm-up, so every call shifts the whole state.  Prints ms per move.  With
--libs A.so B.so ... each library (loaded through EMAP_LIB) is timed in its own process, alternating over --rounds
rounds, and the median per library is reported.  Prints the card, its power limit and SM clocks with the numbers.  Usage: python tools/move_timing.py [--moves N] [--libs LIB ...] [--rounds R]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
SIZES = (1024, 2048)


def _card():
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader",
                            "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        q = "unknown"
    return f"{torch.cuda.get_device_name(0)}; power limit, max SM clock, current SM clock: {q}"


def time_moves(W, moves):
    """ms per move_to of a W x W map (device time between two events on the handle's stream)"""
    import torch
    from elevation_mapping_cupy_b200.elevation_mapping import ElevationMap
    from elevation_mapping_cupy_b200.parameter import core_parameter
    p = core_parameter(W)
    em = ElevationMap(p)
    s = torch.cuda.Stream()
    em.set_stream(s.cuda_stream)
    R = np.eye(3, dtype=np.float32)
    pos = [np.zeros(3), np.array([3 * p.resolution, 2 * p.resolution, 0.0])]
    try:
        with torch.cuda.stream(s):
            for k in range(20):
                em.move_to(pos[k % 2], R)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s)
            for k in range(moves):
                em.move_to(pos[k % 2], R)
            e1.record(s)
        e1.synchronize()
        return e0.elapsed_time(e1) / moves
    finally:
        em.set_stream(None)
        em.close()


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--moves", type=int, default=2000)
    ap.add_argument("--libs", nargs="*", default=None)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", action="store_true", help="one JSON line {W: ms per move} (used with --libs)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("move_timing needs a CUDA device")
    if args.json:
        print(json.dumps({W: time_moves(W, args.moves) for W in SIZES}))
        return
    print(f"card: {_card()}")
    libs = args.libs or [os.environ.get("EMAP_LIB", "")]
    res = {lib: {W: [] for W in SIZES} for lib in libs}
    for _ in range(args.rounds if args.libs else 1):
        for lib in libs:
            env = dict(os.environ, EMAP_LIB=lib) if lib else dict(os.environ)
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--json", "--moves", str(args.moves)],
                                 env=env, capture_output=True, text=True, check=True).stdout
            for W, ms in json.loads(out.strip().splitlines()[-1]).items():
                res[lib][int(W)].append(ms)
    print("| library | map | ms per move (median, min-max over rounds) |")
    print("|---|---|---|")
    for lib in libs:
        for W in SIZES:
            t = np.array(res[lib][W])
            print(f"| {os.path.basename(lib) or 'libemap.so'} | {W}² | {np.median(t):.4f} ({t.min():.4f}-{t.max():.4f}) |",
                  flush=True)


if __name__ == "__main__":
    main()
