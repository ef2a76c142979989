#!/usr/bin/env python
"""Cost of correlating on the device: iso3dfd radius 8 (fp32) at 1024^3, 20 steps, one run_solution(0, 19) call, wall time of the
call and a stream sync:

  none      no correlation (baseline)
  auto      autocorrelation of the whole domain every step (the illumination)
  full      correlation of the whole domain every 5 steps against 4 full-volume rows of a forward solution's recorder, reversed
  snap      correlation of a (2,2,2)-decimated box every step against 20 recorded rows (snapshot imaging)
  loop      `full` done by the host loop: run_solution(t, t), get_elements_in_slice and numpy
  addcmul   torch.Tensor.addcmul_ over three contiguous 1024^3 fp32 tensors, timed by device events: 16 B/point streamed, the
            floor for one correlated frame of `full`
  faces     the six R = 8 faces set every step, from host frames (faces_host) and from a recorder (faces_dev); also the add call

Rounds rotate the order of the forms; each form reports the median of its rounds and the spread (max - min).  The images of
`full` and `loop` must be equal bit for bit, and none, auto, full and snap must leave the same checksum of p.  Each form frees
its solutions before the next, so the peak device memory stays near 48 GB (the forward and adjoint solutions of `full`).  The
card's name, power limit and max SM clock are read (never set) with nvidia-smi in the same run.  Prints one JSON line per form.
"""
import argparse
import json
import statistics
import subprocess
import time

import numpy as np

from yask_b200 import capi
from yask_b200.synth import var_salt

SEED, N, STEPS, R = 7, 1024, 20, 8


def gpu_state():
    try:
        q = "name,power.limit,clocks.max.sm,clocks.sm,temperature.gpu"
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=20).stdout.strip()
    except Exception as e:        # nvidia-smi missing: the numbers stand without it
        return f"unavailable ({e})"


def solution(seed=SEED):
    s = capi.Solution("iso3dfd", radius=R)
    s.set_overall_domain_size_vec((N, N, N))
    s.prepare_solution(0)
    p, v = s.get_var("p"), s.get_var("v")
    for t in (0, 1):
        p.fill_hash(t, seed, var_salt("p", t), -1.0, 1.0)
    v.fill_hash(0, seed, var_salt("v", 0), 0.05, 0.3)
    return s


def timed(s, fn):
    s.sync()
    t0 = time.perf_counter()
    fn()
    s.sync()
    return time.perf_counter() - t0


WHOLE = ([0, 0, 0], [N - 1, N - 1, N - 1])


def forward(rows, every, stride=None):
    """A forward solution that has recorded `rows` rows every `every` steps of the box WHOLE[::stride]."""
    f = solution(SEED + 1)
    f.add_slice("p", *WHOLE, every, rows, stride=stride, every=every)
    f.run_solution(0, STEPS - 1)
    f.sync()
    return f


def form_none(out):
    s = solution()
    ms = timed(s, lambda: s.run_solution(0, STEPS - 1))
    out["checks"].setdefault("p", {})["none"] = s.get_var("p").checksum(STEPS)
    s.close()
    return ms


def form_auto(out):
    s = solution()
    s.add_slice_correlator("p", *WHOLE, 1, STEPS)
    ms = timed(s, lambda: s.run_solution(0, STEPS - 1))
    out["checks"]["p"]["auto"] = s.get_var("p").checksum(STEPS)
    assert s.get_option("slice_correlator_launches") == str(STEPS)
    s.close()
    return ms


def form_full(out):
    f = forward(4, 5)
    s = solution()
    s.add_slice_correlator("p", *WHOLE, 5, 4, src=f, src_id=0, reverse=True, every=5)
    ms = timed(s, lambda: s.run_solution(0, STEPS - 1))
    out["checks"]["p"]["full"] = s.get_var("p").checksum(STEPS)
    img = s.get_correlator_image(0)[0]
    out["checks"]["image_full"] = img.view(np.uint32).astype(np.uint64).sum().item()
    out["images"]["full"] = img
    s.close()
    f.close()
    return ms


def form_snap(out):
    f = forward(STEPS, 1, stride=[2, 2, 2])
    s = solution()
    s.add_slice_correlator("p", *WHOLE, 1, STEPS, src=f, src_id=0, reverse=True, stride=[2, 2, 2])
    ms = timed(s, lambda: s.run_solution(0, STEPS - 1))
    out["checks"]["p"]["snap"] = s.get_var("p").checksum(STEPS)
    s.close()
    f.close()
    return ms


def form_loop(out):
    if "frames" not in out:
        f = forward(4, 5)
        out["frames"] = f.get_slice_frames(0)[0]
        f.close()
    fr = out["frames"]
    s = solution()
    p = s.get_var("p")
    img = np.zeros((N, N, N), np.float32)

    def run():
        for t in range(STEPS):
            s.run_solution(t, t)
            u = t + 1
            if u % 5 == 0:
                box = p.get_elements_in_slice([u] + WHOLE[0], [u] + WHOLE[1])
                np.multiply(box, fr[3 - (u // 5 - 1)], out=box)
                np.add(img, box, out=img)
    ms = timed(s, run)
    s.close()
    out["images"]["loop"] = img
    return ms


def form_addcmul(out):
    import torch
    a = torch.zeros((N, N, N), dtype=torch.float32, device="cuda")
    b = torch.rand((N, N, N), dtype=torch.float32, device="cuda")
    c = torch.rand((N, N, N), dtype=torch.float32, device="cuda")
    a.addcmul_(b, c)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 10
    e0.record()
    for _ in range(reps):
        a.addcmul_(b, c)
    e1.record()
    e1.synchronize()
    ms = e0.elapsed_time(e1) / reps / 1e3
    del a, b, c
    torch.cuda.empty_cache()
    return ms


def faces():
    out = []
    for d in range(3):
        for lo in (True, False):
            f, l = [0, 0, 0], [N - 1] * 3
            if lo:
                l[d] = R - 1
            else:
                f[d] = N - R
            out.append((f, l))
    return out


def form_faces(out, dev):
    fw = solution(SEED + 1)
    for f, l in faces():
        fw.add_slice("p", f, l, 1, STEPS)
    fw.run_solution(0, STEPS - 1)
    host = [fw.get_slice_frames(i)[0] for i in range(6)] if not dev else None
    s = solution()
    t0 = time.perf_counter()
    for i, (f, l) in enumerate(faces()):
        if dev:
            s.add_slice_injector_from("p", f, l, 1, STEPS, fw, i, reverse=True, mode="set")
        else:
            s.add_slice_injector("p", f, l, 1, np.ascontiguousarray(host[i][::-1]), mode="set")
    out["add_call"]["faces_dev" if dev else "faces_host"] = time.perf_counter() - t0
    ms = timed(s, lambda: s.run_solution(0, STEPS - 1))
    out["checks"].setdefault("faces", {})["dev" if dev else "host"] = s.get_var("p").checksum(STEPS)
    s.close()
    fw.close()
    return ms


FORMS = {"none": form_none, "auto": form_auto, "full": form_full, "snap": form_snap, "loop": form_loop, "addcmul": form_addcmul,
         "faces_host": lambda o: form_faces(o, False), "faces_dev": lambda o: form_faces(o, True)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--forms", default=",".join(FORMS))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if capi.device_count() < 1:
        raise SystemExit("bench_slice_correlators: no CUDA device (the engine has no CPU fallback)")
    forms = a.forms.split(",")
    state = {"checks": {"p": {}}, "images": {}, "add_call": {}}
    times = {f: [] for f in forms}
    gpu = gpu_state()
    for r in range(a.rounds):
        order = forms[r % len(forms):] + forms[:r % len(forms)]
        for f in order:
            times[f].append(FORMS[f](state))
    lines = []
    for f in forms:
        t = times[f]
        lines.append({"form": f, "median_s": statistics.median(t), "spread_s": max(t) - min(t), "rounds": t})
    im = state["images"]
    summary = {"gpu": gpu, "n": N, "steps": STEPS,
               "p_checksums_equal": len(set(state["checks"]["p"].values())) == 1,
               "p_checksums": state["checks"]["p"],
               "faces_checksums_equal": len(set(state["checks"].get("faces", {}).values())) <= 1,
               "full_equals_loop": ("full" in im and "loop" in im and np.array_equal(im["full"].view(np.uint32), im["loop"].view(np.uint32))),
               "add_call_s": state["add_call"]}
    med = {x["form"]: x["median_s"] for x in lines}
    if {"none", "full", "addcmul"} <= med.keys():
        summary["full_extra_per_frame_s"] = (med["full"] - med["none"]) / 4
        summary["ratio_to_addcmul"] = summary["full_extra_per_frame_s"] / med["addcmul"]
    text = "\n".join(json.dumps(x) for x in lines + [summary])
    print(text)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
