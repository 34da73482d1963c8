"""Device time of one FNetPlan.run on the headline fnet batch (264 frame pairs of 32x32, bf16) and of each of its launches.

  python tools/ab_fnet.py [--out DIR]

The whole pass and every launch are timed alone in CUDA-graph replay with CUDA events (REPS launches per graph, the
median of ROUNDS replays).  Launches are recorded by wrapping the kernels-module entry points FNetPlan calls, so the tool
measures whichever build of the package it is run from.  Prints the card, its power limit and a table with one row per
launch; DIR/ab_fnet.json gets the same rows.  TECO_PROF_CLIPS / TECO_PROF_LR select another shape."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tecogan_b200 import config, tc_nets, variables as V  # noqa: E402
from tecogan_b200.init_params import xavier_params  # noqa: E402
from tecogan_b200.variables import variable_scope  # noqa: E402

REPS, ROUNDS = 20, 7


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def graph_us(fn):
    """Median device microseconds of one fn() over ROUNDS replays of a graph holding REPS calls."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(REPS):
                fn()
    torch.cuda.current_stream().wait_stream(s)
    g.replay()
    torch.cuda.synchronize()
    ts = []
    for _ in range(ROUNDS):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1000.0 / REPS)
    return sorted(ts)[len(ts) // 2]


def record_launches(plan):
    """[(label, thunk)] of the launches one plan.run() issues, in order."""
    rec = []
    K = tc_nets.K
    wrapped = {}

    def wrap(mod, name, label_fn, restream=False):
        orig = getattr(mod, name)
        wrapped[(mod, name)] = orig

        def f(*a, **kw):
            # a raw `call` ends with the stream it was issued on: the replay takes the stream current then
            thunk = (lambda: orig(*a[:-1], tc_nets.stream_ptr())) if restream else (lambda: orig(*a, **kw))
            rec.append((label_fn(orig, a, kw), thunk))
            return orig(*a, **kw)
        setattr(mod, name, f)

    def conv_label(orig, a, kw):
        x = a[0]
        return "%s %d->%d @ %dx%d" % (orig.__name__, x.shape[-1], kw["cout"], x.shape[1], x.shape[2])

    for name in ("conv3x3_tc", "conv3x3_im2col_tc"):
        if hasattr(K, name):
            wrap(K, name, conv_label)
    wrap(tc_nets, "call", lambda orig, a, kw: a[0], restream=True)
    try:
        plan.run()
        torch.cuda.synchronize()
    finally:
        for (mod, name), orig in wrapped.items():
            setattr(mod, name, orig)
    return rec


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", default=None, help="also write DIR/ab_fnet.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("ab_fnet.py needs a GPU")
    n = int(os.environ.get("TECO_PROF_CLIPS", 264))
    lr = int(os.environ.get("TECO_PROF_LR", 32))
    config.set_precision("bf16")
    V.set_default_store(V.VariableStore()).load(xavier_params(1234, 16))
    with variable_scope('fnet'), variable_scope('autoencode_unit') as fs:
        tc_nets._ensure_vars_fnet()
        plan = tc_nets.FNetPlan(fs, n, lr, lr, "cuda")
    g = torch.Generator().manual_seed(0)
    plan.x_in[..., :6].copy_(torch.rand(n, lr, lr, 6, generator=g).to(torch.bfloat16))
    rec = record_launches(plan)
    whole = graph_us(plan.run)
    rows = [{"launch": i, "what": label, "us": graph_us(fn)} for i, (label, fn) in enumerate(rec)]
    print("card: %s" % card())
    print("FNetPlan.run, %d pairs of %dx%d: %.1f us per pass (%d launches; sum of launches alone %.1f us)" %
          (n, lr, lr, whole, len(rec), sum(r["us"] for r in rows)))
    for r in rows:
        print("  %2d  %-44s %8.1f us" % (r["launch"], r["what"], r["us"]))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "ab_fnet.json"), "w") as f:
            json.dump({"card": card(), "pairs": n, "lr": lr, "pass_us": whole, "launches": rows}, f, indent=1)


if __name__ == "__main__":
    main()
