#!/usr/bin/env python
"""Cost of correlating with a live var of another solution (add_slice_correlator_var) against the snapshot path: iso3dfd radius
8 (fp32) at 1024^3, 20 steps, wall time of the calls and a stream sync:

  adjoint    the adjoint alone, one run_solution(0, 19) call
  alt        G (the reconstruction) and A (the adjoint) alternating one step per call, no correlation: nothing orders the two
             streams, so the runs of G and A may overlap on the device
  alt_linked as alt, with a correlator whose window lies past the run: the same event ordering as a live correlator (each run
             waits for the other solution's last run) and no correlating launch; the baseline of live1 and live5
  live1      as alt, plus a whole-domain correlator of A's p with G's p every step
  live5      as alt, every 5 steps
  snap_f32   the snapshot path: a forward run recording the whole domain every 5 steps (4 rows, float32), then the adjoint with a
             reversed frame correlator; both runs are timed
  snap_bf16  as snap_f32 with bfloat16 frames
  addcmul    torch.Tensor.addcmul_ over three contiguous 1024^3 fp32 tensors, timed by device events: 16 B/point streamed, the
             floor for one correlated frame

Rounds rotate the order of the forms; each form reports the median of its rounds and the spread (max - min).  The summary line
gives the bytes each path holds beyond the adjoint (frames for the snapshot path, one more solution for the live path,
independent of the step count), and a reconstruction check at --acc-n^3 (`accuracy`): F runs 25 steps from zero fields with one
point source; G starts from F's last two steps swapped and re-adds the wavelet reversed, so G.p(u) rebuilds F.p(25 - u); the
relative L2 and max-abs error of G against F's recorded frames is reported per step back (G.p(1) is F.p(24) copied, G.p(2) the
first rebuilt step), and the image of a live correlator against the image of the frame correlator on the same adjoint.  The card's name, power limit and max SM clock are read (never set) with nvidia-smi in the same
run.  Prints one JSON line per form and a summary line.
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


def solution(n=N, seed=SEED, fill=True):
    s = capi.Solution("iso3dfd", radius=R)
    s.set_overall_domain_size_vec((n, n, n))
    s.prepare_solution(0)
    p, v = s.get_var("p"), s.get_var("v")
    if fill:                                  # otherwise p stays zero
        for t in (0, 1):
            p.fill_hash(t, seed, var_salt("p", t), -1.0, 1.0)
    v.fill_hash(0, SEED, var_salt("v", 0), 0.05, 0.3)
    return s


def storage_bytes(s):
    return sum(v.info.storage_bytes for v in s.get_vars())


def timed(sols, fn):
    for s in sols:
        s.sync()
    t0 = time.perf_counter()
    fn()
    for s in sols:
        s.sync()
    return time.perf_counter() - t0


WHOLE = ([0, 0, 0], [N - 1, N - 1, N - 1])


def form_adjoint(out):
    a = solution()
    ms = timed([a], lambda: a.run_solution(0, STEPS - 1))
    a.close()
    return ms


def alternate(g, a):
    for k in range(STEPS):
        g.run_solution(k)
        a.run_solution(k)


def form_alt(out, every=None, linked=False):
    g, a = solution(seed=SEED + 1), solution()
    if every:
        a.add_slice_correlator_var("p", *WHOLE, every, STEPS // every, g, "p", every=every)
    elif linked:
        a.add_slice_correlator_var("p", *WHOLE, STEPS + 1, 1, g, "p", src_t0=1)
    ms = timed([g, a], lambda: alternate(g, a))
    assert a.get_option("slice_correlator_launches") == str(STEPS // every if every else 0)
    out["bytes"]["live_extra_solution"] = storage_bytes(g)
    g.close()
    a.close()
    return ms


def form_snap(out, dtype):
    f, a = solution(seed=SEED + 1), solution()
    f.add_slice("p", *WHOLE, 5, 4, every=5, dtype=dtype)
    a.add_slice_correlator("p", *WHOLE, 5, 4, src=f, src_id=0, reverse=True, every=5)
    ms = timed([f, a], lambda: (f.run_solution(0, STEPS - 1), a.run_solution(0, STEPS - 1)))
    out["bytes"][f"snap_frames_{dtype}"] = 4 * N ** 3 * (4 if dtype == "float32" else 2)
    f.close()
    a.close()
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


FORMS = {"adjoint": form_adjoint, "alt": form_alt, "alt_linked": lambda o: form_alt(o, linked=True), "live1": lambda o: form_alt(o, 1), "live5": lambda o: form_alt(o, 5),
         "snap_f32": lambda o: form_snap(o, "float32"), "snap_bf16": lambda o: form_snap(o, "bfloat16"), "addcmul": form_addcmul}


def ricker(steps, f=0.08, u0=12):
    """The wavelet a(u), u = 1 .. steps: a Ricker of peak frequency f per step centred on step u0."""
    x = (np.pi * f * (np.arange(1, steps + 1) - u0)) ** 2
    return (1 - 2 * x) * np.exp(-x)


def accuracy(n):
    """F runs 25 steps from zero fields with one point source and records p at 5, 10, 15, 20 and at 21 .. 24.  Each F step is
    p(u) = S(p(u-1), p(u-2)) + a(u) with S(x, y) = 2x - y + v lap(x), so p(u-2) = S(p(u-1), p(u)) + a(u): G starts from F's last
    two steps swapped, G.p(0) = F.p(25) and G.p(1) = F.p(24), runs from step 1 (its first run computes G.p(2) from G.p(1) and
    G.p(0)) and adds b(u) = a(27 - u), the wavelet reversed and shifted by one step, so that G.p(u) rebuilds F.p(25 - u).  A runs
    beside G from hash-filled fields with a live correlator on G and a reversed frame correlator on F's frames at 5 .. 20; both
    pair A's step u with F.p(25 - u)."""
    total, every, rows = 25, 5, 4
    box = ([0, 0, 0], [n - 1] * 3)
    centre = [[n // 2, n // 2, n // 2]]
    w = ricker(total)
    f = solution(n, fill=False)
    f.set_sources("p", centre, 1, w[:, None])            # a(u) added to F.p(u), u = 1 .. 25
    f.add_slice("p", *box, every, rows, every=every)      # F.p(5), F.p(10), F.p(15), F.p(20)
    f.add_slice("p", *box, 21, 4)                         # F.p(21) .. F.p(24)
    f.run_solution(0, total - 1)
    fr5, fr1 = f.get_slice_frames(0)[0], f.get_slice_frames(1)[0]
    fp = f.get_var("p")
    g = solution(n, fill=False)
    gp = g.get_var("p")
    gp.set_elements_in_slice(fp.get_elements_in_slice([total] + box[0], [total] + box[1]), [0] + box[0], [0] + box[1])
    gp.set_elements_in_slice(fp.get_elements_in_slice([total - 1] + box[0], [total - 1] + box[1]), [1] + box[0], [1] + box[1])
    g.set_sources("p", centre, 2, w[::-1][:, None])       # b(u) = a(27 - u), u = 2 .. 26
    a = solution(n)
    live = a.add_slice_correlator_var("p", *box, every, rows, g, "p", every=every)
    snap = a.add_slice_correlator("p", *box, every, rows, src=f, src_id=0, reverse=True, every=every)
    err = []

    def compare(u):
        got = gp.get_elements_in_slice([u] + box[0], [u] + box[1]).astype(np.float64)
        want = (fr1[4 - u] if u < every else fr5[(total - u) // every - 1]).astype(np.float64)
        err.append({"g_step": u, "f_step": total - u, "rel_l2": float(np.linalg.norm(got - want) / np.linalg.norm(want)),
                    "max_abs": float(np.abs(got - want).max()), "max_ref": float(np.abs(want).max())})

    compare(1)
    for k in range(total - every):
        if k >= 1:
            g.run_solution(k)
        a.run_solution(k)
        u = k + 1
        if 1 < u < every or u % every == 0:
            compare(u)
    il, isn = (a.get_correlator_image(i)[0].astype(np.float64) for i in (live, snap))
    out = {"n": n, "reconstruction": err, "image_rel_l2_live_vs_snap": float(np.linalg.norm(il - isn) / np.linalg.norm(isn)),
           "image_max_abs_live_vs_snap": float(np.abs(il - isn).max()), "image_max_abs": float(np.abs(isn).max())}
    for s in (f, g, a):
        s.close()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--forms", default=",".join(FORMS))
    ap.add_argument("--acc-n", type=int, default=512, help="domain edge of the reconstruction check (0: skip it)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if capi.device_count() < 1:
        raise SystemExit("bench_slice_correlators_var: no CUDA device (the engine has no CPU fallback)")
    forms = a.forms.split(",")
    state = {"bytes": {}}
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
    med = {x["form"]: x["median_s"] for x in lines}
    summary = {"gpu": gpu, "n": N, "steps": STEPS, "bytes": state["bytes"]}
    if {"alt_linked", "live1"} <= med.keys():
        summary["live_per_frame_s"] = (med["live1"] - med["alt_linked"]) / STEPS
    if {"alt_linked", "live5"} <= med.keys():
        summary["live5_per_frame_s"] = (med["live5"] - med["alt_linked"]) / (STEPS // 5)
    for f in ("alt", "alt_linked"):
        if {f, "adjoint"} <= med.keys():
            summary[f"{f}_over_two_adjoints_s"] = med[f] - 2 * med["adjoint"]
    if "addcmul" in med and "live_per_frame_s" in summary:
        summary["live_ratio_to_addcmul"] = summary["live_per_frame_s"] / med["addcmul"]
    if a.acc_n:
        summary["accuracy"] = accuracy(a.acc_n)
    text = "\n".join(json.dumps(x) for x in lines + [summary])
    print(text)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
