"""Shared helpers for the parity tests: run the same model directory + inputs through two libraries exporting the
reference's C ABI (the engine and the reference-compiled oracle) and compare every requested tensor.

The reference's outputs are stored under tests/golden/oracle/, keyed by a hash of what determines them (model text, inputs,
options), so the suite needs no reference build: `reference_outputs` / `stored_reference` read the stored result and run the oracle
library only when no result is stored.  With OSB_GOLDEN_RECORD=<dir> every result computed by the oracle is also written to <dir>
(copy the files to tests/golden/oracle/ to commit them).  Floating-point tensors above SAMPLE_ABOVE elements are stored as a fixed
seeded sample of SAMPLE elements (`Sampled`); `report` compares a full tensor with such a sample at the sampled positions.  Integer
tensors are stored whole (the uint8 tests compare them bit for bit)."""
import hashlib
import os

import numpy as np
import pytest

from onnxstream_b200.model import Model

GOLDEN_ORACLE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "oracle")
SAMPLE_ABOVE = 1024
SAMPLE = 512
# The sampled positions are the first SAMPLE of a seeded draw of SAMPLE_DRAW positions.  The draw size is part of the stored format:
# numpy's draw of 2048 and its draw of 512 pick different positions, and the stored samples were taken at these ones.
SAMPLE_DRAW = 2048


class Sampled:
    """A stored reference tensor reduced to the values at fixed flat positions `idx`."""

    def __init__(self, shape, idx, values):
        self.shape, self.idx, self.values = tuple(int(x) for x in shape), idx, values
        self.size = int(np.prod(self.shape))

    def __array__(self, dtype=None, copy=None):
        raise TypeError("a sampled reference tensor supports shape and report() only")


def _sample_idx(size):
    """The first SAMPLE of a fixed seeded draw of min(size, SAMPLE_DRAW) distinct flat positions, sorted."""
    draw = np.random.default_rng(size).choice(size, min(size, SAMPLE_DRAW), replace=False)
    return np.sort(draw[:SAMPLE]).astype(np.int64)


def _key(parts):
    h = hashlib.sha1()
    for p in parts:
        if isinstance(p, dict):
            for k in sorted(p):
                v = np.ascontiguousarray(p[k])
                h.update(k.encode()); h.update(str(v.dtype).encode()); h.update(repr(v.shape).encode()); h.update(v.tobytes())
        elif isinstance(p, bytes):
            h.update(p)
        else:
            h.update(repr(p).encode())
    return h.hexdigest()


def _save(fn, out, whole=False):
    arrays = {"__names__": np.array(sorted(out), dtype=object).astype(str)}
    for n, v in out.items():
        if v is None:
            continue
        v = np.asarray(v)
        if not whole and v.size > SAMPLE_ABOVE and v.dtype.kind == "f":
            idx = _sample_idx(v.size)
            arrays["s/" + n] = np.array(v.shape, np.int64)
            arrays["d/" + n] = np.diff(idx, prepend=0).astype(np.int32)     # sorted positions, delta-encoded (compresses well)
            arrays["v/" + n] = v.reshape(-1)[idx]
        else:
            arrays["v/" + n] = v
    os.makedirs(os.path.dirname(fn), exist_ok=True)
    np.savez_compressed(fn, **arrays)


def _load(fn):
    z = np.load(fn)
    out = {}
    for n in z["__names__"]:
        n = str(n)
        if "v/" + n not in z:
            out[n] = None
        elif "s/" + n in z:
            out[n] = Sampled(z["s/" + n], np.cumsum(z["d/" + n].astype(np.int64)), z["v/" + n])
        else:
            out[n] = z["v/" + n]
    return out


def stored_reference(key_parts, compute, whole=False):
    """The reference result identified by key_parts: the stored one, else compute() (which runs the oracle library).
    whole=True: recorded without sampling, for tests that compare tensors element for element."""
    key = _key(key_parts)
    fn = os.path.join(GOLDEN_ORACLE, key + ".npz")
    if os.path.exists(fn):
        return _load(fn)
    out = compute()
    rec = os.environ.get("OSB_GOLDEN_RECORD")
    if rec:
        _save(os.path.join(rec, key + ".npz"), out, whole)
    return out


def model_text(model_dir):
    with open(model_dir.rstrip("/") + "/model.txt", "rb") as f:
        return f.read()


def reference_outputs(oracle_lib, model_dir, inputs, options=(), whole=False, **kw):
    """run_model(oracle_lib, ...)[0], served from tests/golden/oracle when stored (whole: see stored_reference)."""
    def compute():
        if oracle_lib is None:
            pytest.fail("no stored reference output for this case and no oracle library (oracle/_ref/liboracle_ref.so) to compute it")
        return run_model(oracle_lib, model_dir, inputs, options, **kw)[0]
    return stored_reference((model_text(model_dir), inputs, tuple(options), sorted(kw.items())), compute, whole)


def run_model(lib, model_dir, inputs, options=(), extra_outputs=(), wp="nocache", parts=None, ranges=None, upcast=(), b200_options=(), runs=1, plain_abi=False):
    m = Model(lib, 4, wp, plain_abi=plain_abi)   # 4 pthreadpool workers for the CPU oracle (0 = every core: slow on many-core hosts); the GPU engine ignores it
    for o in options:
        m.set_option(o, True)
    for name, val in b200_options:
        m.lib.model_set_option(m.h, name.encode(), int(val))
    if parts is not None:
        m.set_attention_parts(parts)
    for k, (mn, mx) in (ranges or {}).items():
        m.set_range(k, mn, mx)
    for p in upcast:
        m.add_upcast_pattern(p)
    for e in extra_outputs:
        m.add_extra_output(e)
    m.read_file(model_dir.rstrip("/") + "/model.txt")
    out = None
    for _ in range(runs):
        m.clear_tensors()
        for k, v in inputs.items():
            m.add_tensor(k, v)
        m.run()
        out = {}
        for n in m.get_all_tensor_names():
            t = m.get_tensor(n)
            if t is None and not plain_abi:
                t = m.get_tensor_i64(n)
            out[n] = t
    return out, m


def report(a, b):
    if isinstance(a, Sampled) and isinstance(b, Sampled):
        assert a.shape == b.shape and np.array_equal(a.idx, b.idx)
        a, b = a.values, b.values
    elif isinstance(b, Sampled):
        a, b = np.asarray(a).reshape(-1)[b.idx], b.values
    elif isinstance(a, Sampled):
        a, b = a.values, np.asarray(b).reshape(-1)[a.idx]
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    d = np.abs(a - b)
    denom = max(np.abs(b).max(), 1e-12)
    return dict(max_abs=float(d.max()) if d.size else 0.0, rel_to_max=float(d.max() / denom) if d.size else 0.0,
                rms=float(np.sqrt((d ** 2).mean())) if d.size else 0.0, ref_rms=float(np.sqrt((b ** 2).mean())) if b.size else 0.0)
