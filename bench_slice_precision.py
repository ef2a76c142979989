#!/usr/bin/env python
"""Cost and accuracy of narrowed frames and double images: iso3dfd radius 8 (fp32) at 1024^3, 20 steps, one run_solution(0, 19)
call, wall time of the call and a stream sync:

  none           no slices (baseline)
  rec_<F>        a full-volume recorder every 5 steps (4 rows), frames in F = f32, bf16, f16
  cor_<F>_<I>    the adjoint: whole-domain correlation every 5 steps against those 4 rows of a forward solution, reversed, with
                 an image in I = f32, f64
  auto_<I>       whole-domain autocorrelation every step, image in I
  addcmul        torch.Tensor.addcmul_ over three contiguous 1024^3 fp32 tensors, timed by device events: the 16 B/point floor
                 of one correlated frame with f32 frames and image

Bytes streamed per point of one recorded or correlated frame: recorder 8 B (read var, write an f32 frame), 6 B with 16-bit
frames; correlator 16 B (read var, read frame, read and write the image), 14 B with 16-bit frames, 24 B with a double image.

Rounds rotate the order of the forms; each form reports the median of its rounds and the spread (max - min).  The recorders
must leave p's checksum equal to the baseline's.  Accuracy (first round): the relative L2 and max-abs difference of the cor
images, 16-bit frames against f32 frames with the same image type, and f32 images against f64 images with the same frames,
over every 8th x plane (134M points).  Capacity: full-volume frames of each type that fit in cudaMemGetInfo's free memory after
one solution is prepared, less a 2 GiB margin -- computed, never allocated.  The card's name, power limit and max SM clock are
read (never set) with nvidia-smi in the same run.  Prints one JSON line per form and a summary line.
"""
import argparse
import json
import statistics
import time

import numpy as np

from bench_slice_correlators import N, STEPS, WHOLE, form_addcmul, gpu_state, solution, timed
from yask_b200 import capi

EVERY, ROWS = 5, 4
FRAMES = {"f32": "float32", "bf16": "bfloat16", "f16": "float16"}
IMAGES = {"f32": "float32", "f64": "float64"}


def form_none(st):
    s = solution()
    t = timed(s, lambda: s.run_solution(0, STEPS - 1))
    st["checks"]["none"] = s.get_var("p").checksum(STEPS)
    s.close()
    return t


def form_rec(st, f):
    s = solution()
    s.add_slice("p", *WHOLE, EVERY, ROWS, every=EVERY, dtype=FRAMES[f])
    t = timed(s, lambda: s.run_solution(0, STEPS - 1))
    st["checks"][f"rec_{f}"] = s.get_var("p").checksum(STEPS)
    assert s.get_option("slice_launches") == str(ROWS)
    s.close()
    return t


def form_cor(st, f, i):
    fw = solution(8)
    fw.add_slice("p", *WHOLE, EVERY, ROWS, every=EVERY, dtype=FRAMES[f])
    fw.run_solution(0, STEPS - 1)
    fw.sync()
    s = solution()
    s.add_slice_correlator("p", *WHOLE, EVERY, ROWS, src=fw, src_id=0, reverse=True, every=EVERY, image_dtype=IMAGES[i])
    t = timed(s, lambda: s.run_solution(0, STEPS - 1))
    assert s.get_option("slice_correlator_launches") == str(ROWS)
    key = f"cor_{f}_{i}"
    if key not in st["images"]:
        st["images"][key] = np.ascontiguousarray(s.get_correlator_image(0)[0][::8], np.float64)
    s.close()
    fw.close()
    return t


def form_auto(st, i):
    s = solution()
    s.add_slice_correlator("p", *WHOLE, 1, STEPS, image_dtype=IMAGES[i])
    t = timed(s, lambda: s.run_solution(0, STEPS - 1))
    assert s.get_option("slice_correlator_launches") == str(STEPS)
    s.close()
    return t


def capacity():
    """Full-volume frames of each type that fit beside one prepared solution, with a 2 GiB margin."""
    import torch
    s = solution()
    s.sync()
    free, total = torch.cuda.mem_get_info()
    s.close()
    room = free - (2 << 30)
    return {"free_bytes": free, "total_bytes": total,
            "frames": {f: room // (N ** 3 * (4 if f == "f32" else 2)) for f in FRAMES}}


def diff(a, ref):
    d = a - ref
    return {"rel_l2": float(np.linalg.norm(d) / np.linalg.norm(ref)), "max_abs": float(np.abs(d).max()),
            "ref_max_abs": float(np.abs(ref).max())}


FORMS = {"none": form_none, "addcmul": form_addcmul}
FORMS.update({f"rec_{f}": (lambda st, f=f: form_rec(st, f)) for f in FRAMES})
FORMS.update({f"cor_{f}_{i}": (lambda st, f=f, i=i: form_cor(st, f, i)) for f in FRAMES for i in IMAGES})
FORMS.update({f"auto_{i}": (lambda st, i=i: form_auto(st, i)) for i in IMAGES})


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--forms", default=",".join(FORMS))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if capi.device_count() < 1:
        raise SystemExit("bench_slice_precision: no CUDA device (the engine has no CPU fallback)")
    forms = a.forms.split(",")
    st = {"checks": {}, "images": {}}
    times = {f: [] for f in forms}
    gpu = gpu_state()
    cap = capacity()
    for r in range(a.rounds):
        order = forms[r % len(forms):] + forms[:r % len(forms)]
        for f in order:
            t0 = time.perf_counter()
            times[f].append(FORMS[f](st))
            print(f"# round {r} {f}: {times[f][-1]:.4f} s ({time.perf_counter() - t0:.1f} s with set-up)", flush=True)
    lines = [{"form": f, "median_s": statistics.median(t), "spread_s": max(t) - min(t), "rounds": t} for f, t in times.items()]
    med = {x["form"]: x["median_s"] for x in lines}
    im = st["images"]
    acc = {}
    for i in IMAGES:
        for f in ("bf16", "f16"):
            if f"cor_{f}_{i}" in im and f"cor_f32_{i}" in im:
                acc[f"{f}_vs_f32_frames_image_{i}"] = diff(im[f"cor_{f}_{i}"], im[f"cor_f32_{i}"])
    for f in FRAMES:
        if f"cor_{f}_f32" in im and f"cor_{f}_f64" in im:
            acc[f"f32_vs_f64_image_frames_{f}"] = diff(im[f"cor_{f}_f32"], im[f"cor_{f}_f64"])
    summary = {"gpu": gpu, "n": N, "steps": STEPS, "capacity": cap, "accuracy": acc,
               "p_checksums": st["checks"], "p_checksums_equal": len(set(st["checks"].values())) <= 1}
    if "none" in med:
        summary["per_frame_s"] = {f: (med[f] - med["none"]) / ROWS for f in med if f.startswith(("rec_", "cor_"))}
        summary["per_frame_s"].update({f: (med[f] - med["none"]) / STEPS for f in med if f.startswith("auto_")})
        if "addcmul" in med:
            summary["per_frame_over_addcmul"] = {f: v / med["addcmul"] for f, v in summary["per_frame_s"].items()}
    text = "\n".join(json.dumps(x) for x in lines + [summary])
    print(text)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
