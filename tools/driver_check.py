"""Render the same calls through two (or more) builds of libcrgpu.so and compare what they enqueue and compute.

Each library runs in its own child process (tests/test_gpu_launch_schedule.py's call shapes: rectangles and tile sets that fit,
overlap or need pieces, armed and unarmed, no bounces, FLAG_COUNT, FLAG_TIME_KERNELS, and armed calls with the stop already
requested) with no CRGPU_* variable set.  Every shape prints kernel_launches, paths, rays and the framebuffer's CRC32; the check
passes when every library gives the same line for every shape.  The card's name and power limit are read in the same run.

    python tools/driver_check.py LIB [LIB ...] [--out profiles/r04_driver_check.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "c-ray_b200"), os.path.join(ROOT, "tests")]

import test_gpu_launch_schedule as S  # noqa: E402


def smi(fields):
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader"], stdout=subprocess.PIPE, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unavailable: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="+")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    out = {"card": smi("name,power.limit"), "libs": [os.path.relpath(os.path.abspath(p), ROOT) for p in args.libs], "shapes": {}}
    runs = [S.run_child(os.path.abspath(p)) for p in args.libs]
    same = True
    for name in S.SHAPES:
        recs = [r.get(name) for r in runs]
        match = all(rec == recs[0] for rec in recs)
        same &= match
        out["shapes"][name] = {"records": recs, "match": match}
        print(json.dumps({"shape": name, "match": match, "records": recs}), flush=True)
    out["all_match"] = same
    text = json.dumps(out, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(text + "\n")
    print("ALL MATCH" if same else "MISMATCH")
    sys.exit(0 if same else 1)


if __name__ == "__main__":
    main()
