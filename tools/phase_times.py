"""Serialised per-phase wall times of one C4 training step (each phase followed by a device sync), with the
option-stream overlap off and on.  Diagnostic only: the sum is NOT the step time (phases overlap in the real step)."""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def run(overlap):
    from bench import headline_params
    from visdial_b200 import Batch, Model
    from visdial_b200.synthetic import make_batch
    p = headline_params(0)
    p["batchSize"] = 32
    model = Model(p, seed=1)
    eng = model.engine
    eng.set_option_overlap(overlap)
    batch = Batch(make_batch(p, 32, seed=5)).to_device(eng)
    phases = ["zero", "enc_fwd", "dec_fwd", "crit_fwd", "crit_bwd", "dec_bwd", "bconn", "enc_bwd", "adam"]
    acc = {k: 0.0 for k in phases}
    steps = 8
    for it in range(steps + 2):
        t = {}

        def tick(name, fn):
            t0 = time.perf_counter()
            r = fn()
            eng.synchronize()
            t[name] = (time.perf_counter() - t0) * 1e3
            return r
        tick("zero", eng.zero_grad)
        tick("enc_fwd", lambda: eng.encoder_forward(batch))
        tick("dec_fwd", lambda: eng.decoder_forward(batch))
        tick("crit_fwd", lambda: eng.criterion_forward(batch))
        tick("crit_bwd", lambda: eng.criterion_backward(batch))
        tick("dec_bwd", lambda: eng.decoder_backward(batch))
        g = tick("bconn", lambda: eng.backward_connect(batch))
        tick("enc_bwd", lambda: eng.encoder_backward(batch, g))
        tick("adam", lambda: eng.clamp_adam_step(1e-3))
        if it >= 2:
            for k in phases:
                acc[k] += t[k] / steps
    print("overlap=%d " % overlap + " ".join("%s=%.2f" % (k, acc[k]) for k in phases) + " sum=%.2f" % sum(acc.values()), flush=True)
    eng.close()


if __name__ == "__main__":
    run(int(sys.argv[1]) if len(sys.argv) > 1 else 0)
