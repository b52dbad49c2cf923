#!/usr/bin/env python
"""Where the time of the TMA ring kernels goes at 512^3 fp64 on one GPU: the fused forward t0 (fft_tma_fused_zy_kernel) and
the forward X pass (fft_tma_pass_kernel<TMA_XF>) (developer tool).

    python distributedfft_b200/csrc/tools/t0_profile.py [--lag 3 --lag 4 ...] [--reps 20] [--rounds 3] [--out DIR]

Builds t0_profile.cu (the kernel bodies as the library instantiates them at C = 8 and C = 4, their movement-only twins and
stamped variants, the X pass's pre-mover structure without arithmetic, and a plain TMA copy of the slab) against libdfft.so
(run `python -m distributedfft_b200.build` first) into a temporary directory, runs it and prints one JSON object:
  - the card's name, power limit and SM clock (nvidia-smi, read-only query) before and after;
  - ms per launch of every variant, per round (the rounds alternate the variants), and per variant the min and max;
  - from one stamped launch of each ring kernel (the fused kernel and its twin at the first lag), per role (Z, Y; the X
    pass is all role Z): median and p90 in microseconds of
      load_wait     the consumer group waiting for the slot to land (TMS_FULL - TMS_READY)
      dep_wait      mover waiting for the plane counter (TMS_DEP - TMS_TICKET; 0 for Z tiles)
      load_latency  load issued to the consumers taking the slot (TMS_FULL - TMS_LOAD)
      transform     slot full to transform done (TMS_DONE - TMS_FULL)
      store_read    store issued to the store having read the slot, which frees it (TMS_FREED - TMS_STORE)
      store_retire  store issued to complete and published (TMS_RETIRED - TMS_STORE; other tiles: to their slot freed)
    and the ring occupancy: the mean number of tiles a CTA holds in each state over the launch (time in state / span), and the
    share of the span in which its consumer groups wait for a load (summed over groups).
The stamps are %globaltimer values; the tick the card shows is printed as `timer_tick_ns`."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(os.path.dirname(HERE))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

WHO, TICKET, DEP, LOAD, READY, FULL, DONE, STORE, FREED, RETIRED, NSTAMP = range(11)   # TMS_* in fft_tma.cuh


def gpu_state():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        name, plim, clk, mx = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": plim, "sm_clock": clk, "max_sm_clock": mx}
    except Exception as exc:   # the numbers still stand; the record says why the card state is missing
        return {"error": str(exc)}


def build(tmp):
    exe = os.path.join(tmp, "t0_profile")
    cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-ccbin", "/usr/bin/g++",
           os.path.join(HERE, "t0_profile.cu"), "-o", exe, "-L", PKG, "-ldfft", "-Xlinker", "-rpath", "-Xlinker", PKG]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.exit("build failed:\n" + r.stdout + r.stderr)
    return exe


def stats(x):
    import numpy as np
    if len(x) == 0:
        return None
    return {"median_us": round(float(np.median(x)) / 1e3, 3), "p90_us": round(float(np.percentile(x, 90)) / 1e3, 3)}


def analyse(path):
    import numpy as np
    s = np.fromfile(path, dtype=np.uint64).reshape(-1, NSTAMP).astype(np.int64)
    if (s[:, TICKET:] == 0).any():
        sys.exit(f"{path}: some tickets carry no stamps")
    t0 = s[:, TICKET].min()
    span = s[:, RETIRED].max() - t0
    y = (s[:, WHO] & 1).astype(bool)
    cta = s[:, WHO] >> 1
    ncta = int(cta.max()) + 1
    d = {
        "load_wait": s[:, FULL] - s[:, READY],
        "dep_wait": s[:, DEP] - s[:, TICKET],
        "load_latency": s[:, FULL] - s[:, LOAD],
        "transform": s[:, DONE] - s[:, FULL],
        "store_read": s[:, FREED] - s[:, STORE],
        "store_retire": s[:, RETIRED] - s[:, STORE],
    }
    out = {"span_ms": round(span / 1e6, 4)}
    for role, m in (("Z", ~y), ("Y", y)):
        if m.any():
            out[role] = {k: stats(v[m]) for k, v in d.items()}
    # mean tiles per CTA in each state (Little's law: total time in the state / span / CTAs)
    states = {
        "dep_wait": (TICKET, DEP), "issued_to_taken": (LOAD, FULL), "transforming": (FULL, DONE),
        "done_to_store": (DONE, STORE), "store_to_freed": (STORE, FREED), "held": (TICKET, FREED),
    }
    occ = {}
    for k, (a, b) in states.items():
        tot = (s[:, b] - s[:, a]).sum()
        occ[k] = round(float(tot) / span / ncta, 3)
    occ["consumer_waiting_share"] = round(float(d["load_wait"].sum()) / span / ncta, 3)
    out["ring_occupancy"] = occ
    diffs = np.diff(np.unique(s[:, TICKET:RETIRED + 1].ravel()))
    out["timer_tick_ns"] = int(diffs[diffs > 0].min()) if len(diffs) else None
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lag", type=int, action="append")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", help="keep the stamp files here (default: a temporary directory)")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        exe = build(tmp)
        out = args.out or tmp
        os.makedirs(out, exist_ok=True)
        before = gpu_state()
        cmd = [exe, "--out", out, "--reps", str(args.reps), "--rounds", str(args.rounds)]
        for lag in args.lag or [3]:
            cmd += ["--lag", str(lag)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        after = gpu_state()
        if r.returncode != 0:
            sys.exit("t0_profile failed:\n" + r.stdout + r.stderr)
        res = json.loads(r.stdout)
        res["gpu_before"], res["gpu_after"] = before, after
        names = res["rounds"][0].keys()
        res["spread"] = {k: [min(r[k] for r in res["rounds"]), max(r[k] for r in res["rounds"])] for k in names}
        for st in res["stamped"]:
            res["profile_" + st["name"]] = analyse(os.path.join(out, "stamps_%s.bin" % st["name"]))
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
