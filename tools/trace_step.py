"""Device timeline of one benched training step (C4 by default: mn-att-ques-im-hist + disc, B = 32, VD_MATH_F16, option
stream overlapped), recorded with torch.profiler (CUDA activities) after warm-up.

Writes to --out:
  step<i>.json   the Chrome trace of profiled step i (open in chrome://tracing or Perfetto)
  summary.txt    what is printed: per stream, the busy intervals by kernel name; the phases of the option stream
                 (forward and BPTT steps, fp16 weight gradient, token sort, segmented sum, dP contractions, colsum);
                 the grid of each persistent launch; and where the option stream's tail ends against the other streams

usage: python tools/trace_step.py [--out DIR] [--steps 3] [--warmup 3] [--config C4] [--batch 32]"""
import argparse
import collections
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# option-stream phases, by kernel-name substring (first match wins)
PHASES = [("opt_fwd_step", "k_lstm16<0>"), ("opt_fwd_first", "k_lstm16_first"), ("opt_bptt_step", "k_lstm16_bptt"),
          ("opt_bptt_last", "k_lstm16_bwd_last"), ("wgrad_atb16", "k_atb16"), ("token_sort", "k_tok_"),
          ("segsum16", "k_segsum16"), ("colsum", "colsum"), ("dP_gemm", "k_tc_"), ("dP_gemm", "gemm")]
PERSISTENT = ("k_lstm16<", "k_lstm16_bptt", "k_atb16", "k_enc_pair")


def short(name):
    n = name.split("(")[0]
    return n.replace("void ", "").replace("vd::tc::", "").replace("vd::", "").strip()


def phase_of(name):
    for ph, key in PHASES:
        if key in name:
            return ph
    return "other"


def kernels(trace_path):
    with open(trace_path) as f:
        ev = json.load(f)["traceEvents"]
    ks = [e for e in ev if e.get("cat") == "kernel" and "dur" in e]
    t0 = min(e["ts"] for e in ks)
    out = []
    for e in ks:
        a = e.get("args", {})
        out.append(dict(name=e["name"], s=(e["ts"] - t0) / 1e3, e=(e["ts"] + e["dur"] - t0) / 1e3, stream=a.get("stream", -1),
                        grid=tuple(a.get("grid", ())), block=tuple(a.get("block", ()))))
    return sorted(out, key=lambda k: k["s"])


def runs(ks):
    """consecutive launches of the same kernel on one stream merged into one busy interval"""
    out = []
    for k in ks:
        n = short(k["name"])
        if out and out[-1][0] == n:
            out[-1][2] = k["e"]; out[-1][3] += 1; out[-1][4] += k["e"] - k["s"]
        else:
            out.append([n, k["s"], k["e"], 1, k["e"] - k["s"]])
    return out


def analyse(ks, lines, verbose):
    by_stream = collections.defaultdict(list)
    for k in ks:
        by_stream[k["stream"]].append(k)
    opt = max(by_stream, key=lambda s: sum(1 for k in by_stream[s] if "k_lstm16_bptt" in k["name"]))
    step_end = max(k["e"] for k in ks)
    r = {"step_ms": step_end}
    if verbose:
        for s, sk in sorted(by_stream.items(), key=lambda kv: kv[1][0]["s"]):
            busy = sum(k["e"] - k["s"] for k in sk)
            lines.append("stream %s%s: %d kernels, busy %.3f ms, %.3f .. %.3f ms" %
                         (s, " (option stream)" if s == opt else "", len(sk), busy, sk[0]["s"], sk[-1]["e"]))
            for n, a, b, c, d in runs(sk):
                if d >= 0.02 or c > 1:
                    lines.append("    %8.3f .. %8.3f  %7.3f busy  x%-4d %s" % (a, b, d, c, n))
    # option-stream phases: span and busy time
    ph = collections.OrderedDict()
    for k in by_stream[opt]:
        p = phase_of(k["name"])
        q = ph.setdefault(p, [k["s"], k["e"], 0.0, 0])
        q[0] = min(q[0], k["s"]); q[1] = max(q[1], k["e"]); q[2] += k["e"] - k["s"]; q[3] += 1
    for p, (a, b, d, c) in ph.items():
        r["opt." + p] = d
    bptt_end = max((k["e"] for k in by_stream[opt] if "k_lstm16_bptt" in k["name"]), default=0.0)
    opt_end = by_stream[opt][-1]["e"]
    r["opt_tail_ms"] = opt_end - bptt_end          # last BPTT step -> last kernel of the option stream
    # the other streams' last kernel that ends before the option stream does, and who waits for the option stream
    others = [k for k in ks if k["stream"] != opt]
    enc_before = max((k["e"] for k in others if k["e"] <= opt_end), default=0.0)
    after = [k for k in others if k["s"] >= opt_end - 1e-3]
    nxt = min((k["s"] for k in after), default=opt_end)
    r["others_last_end_before_opt_end_ms"] = enc_before
    r["exposed_tail_ms"] = max(0.0, opt_end - enc_before)
    if verbose:
        lines.append("option stream phases (span / busy ms, launches):")
        for p, (a, b, d, c) in ph.items():
            lines.append("    %-14s %8.3f .. %8.3f  busy %7.3f  x%d" % (p, a, b, d, c))
        lines.append("grids of the persistent launches:")
        seen = collections.Counter()
        for k in ks:
            if any(p in k["name"] for p in PERSISTENT):
                seen[(short(k["name"]), k["grid"], k["stream"])] += 1
        for (n, g, s), c in sorted(seen.items()):
            lines.append("    %-28s grid %-14s stream %s  x%d" % (n, g, s, c))
        lines.append("last BPTT step ends %.3f ms; option stream ends %.3f ms (tail %.3f ms)" % (bptt_end, opt_end, r["opt_tail_ms"]))
        lines.append("other streams: last kernel ending before that %.3f ms; next kernel after it starts %.3f ms" % (enc_before, nxt))
        lines.append("=> the option tail %s the critical path: the other streams sit idle for %.3f ms waiting for it" %
                     ("IS on" if r["exposed_tail_ms"] > 0.05 else "is NOT on", r["exposed_tail_ms"]))
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="trace_out")
    ap.add_argument("--config", default="C4")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    import bench
    from visdial_b200 import VD_MATH_F16, Batch, Model
    from visdial_b200.synthetic import make_batch

    os.makedirs(a.out, exist_ok=True)
    p = bench.config_params(a.config)
    p["batchSize"] = a.batch
    m = Model(p, seed=1234)
    eng = m.engine
    eng.set_math_mode(VD_MATH_F16)
    eng.set_option_overlap(True)
    b = Batch(make_batch(p, a.batch, seed=1234)).to_device(eng)

    class L:
        def getTrainBatch(self, params):
            return b

    for _ in range(a.warmup):
        m.trainIteration(L())
    eng.synchronize()
    lines = ["%s, %s, %s" % (a.config, torch.cuda.get_device_name(0), "B = %d" % a.batch)]
    res = []
    for i in range(a.steps):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            m.trainIteration(L())
            eng.synchronize()
        path = os.path.join(a.out, "step%d.json" % i)
        prof.export_chrome_trace(path)
        ks = kernels(path)
        if not ks:
            raise SystemExit("the profiler recorded no kernels of the library")
        if i == a.steps - 1:
            lines.append("---- step %d" % i)
        res.append(analyse(ks, lines, i == a.steps - 1))
    lines.append("---- median over %d profiled steps (ms)" % a.steps)
    for k in res[0]:
        vals = [r.get(k, 0.0) for r in res]
        lines.append("    %-36s %8.3f   (min %.3f, max %.3f)" % (k, statistics.median(vals), min(vals), max(vals)))
    text = "\n".join(lines)
    print(text)
    with open(os.path.join(a.out, "summary.txt"), "w") as f:
        f.write(text + "\n")


if __name__ == "__main__":
    main()
