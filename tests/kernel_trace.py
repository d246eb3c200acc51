"""The kernels one eager engine run launches, from a torch.profiler trace taken in a child process.

A profiler session leaves CUDA activity tracing set up in the process that ran it, and a later session in the same process can lose the
first part of its trace (more so the more kernels ran in between).  Tracing in a child process keeps every test's trace whole, whatever
ran before it."""
import json
import os
import subprocess
import sys

import numpy as np

TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)

_CHILD = """
import json, sys
import numpy as np
sys.path[:0] = [%r, %r]
import torch
from torch.profiler import ProfilerActivity, profile
from util import run_model
lib, d, spec = sys.argv[1], sys.argv[2], json.load(open(sys.argv[3]))
inputs = dict(np.load(d + "/trace_inputs.npz"))
torch.cuda.init()
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    out, _ = run_model(lib, d, inputs, spec["options"], extra_outputs=spec["extra"], wp=spec["wp"], b200_options=[tuple(o) for o in spec["b200"]])
    torch.cuda.synchronize()
evs = sorted((e for e in prof.events() if e.device_type.name == "CUDA"), key=lambda e: e.time_range.start)
np.savez(d + "/trace_out.npz", **{k: np.asarray(v) for k, v in out.items() if k in spec["keep"]})
json.dump([e.name for e in evs], open(d + "/trace_kernels.json", "w"))
""" % (ROOT, TESTS)


def trace_run(lib, d, inputs, options=(), extra_outputs=(), keep=(), wp="nocache", b200_options=()):
    """Runs the model in directory d once, eagerly, in a child process: (the outputs named in `keep`, kernel names in launch order)."""
    np.savez(os.path.join(d, "trace_inputs.npz"), **inputs)
    spec = os.path.join(d, "trace_spec.json")
    with open(spec, "w") as f:
        json.dump({"options": list(options), "extra": list(extra_outputs), "keep": list(keep), "wp": wp, "b200": [list(o) for o in b200_options]}, f)
    r = subprocess.run([sys.executable, "-c", _CHILD, lib, d, spec], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    out = dict(np.load(os.path.join(d, "trace_out.npz")))
    with open(os.path.join(d, "trace_kernels.json")) as f:
        return out, json.load(f)
