"""2-GPU parity (skips with < 2 GPUs): the NCCL weight-distribution paths of the WeightStreamer, checked on EVERY rank against the
reference's CPU path -- rank 0 is the root that never receives data, so rank 1's output is the one that proves the collective."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from onnxstream_b200 import emit
from util import reference_outputs

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ngpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.skipif(_ngpus() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("sharded", ["1", "0"])
def test_two_ranks_match_reference(oracle_lib, sharded):
    with tempfile.TemporaryDirectory(prefix="osb200_mgpu_") as tmp:
        d = tmp + "/"
        cfg = emit.UNetConfig.tiny(16)
        emit.emit_unet(d, cfg, "float16", seed=0)
        # each rank's reference output (sample seed = rank), handed to the workers as files
        for r in range(2):
            ref = reference_outputs(oracle_lib, d, emit.unet_inputs(cfg, seed=r), ("use_fp16_arithmetic", "fuse_ops_in_attention"))
            np.save(os.path.join(tmp, f"ref{r}.npy"), ref["out_5F_sample"])
        env = dict(os.environ, OSB_SHARDED_H2D=sharded)
        env.pop("CUDA_VISIBLE_DEVICES", None)
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", "29613",
               os.path.join(ROOT, "tests", "mgpu_worker.py"), d, tmp]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600, env=env)
        lines = [l for l in r.stdout.splitlines() if l.startswith("MGPU_")]
        assert r.returncode == 0 and len(lines) == 2 and all(l.startswith("MGPU_OK") for l in lines), r.stdout[-3000:]
        assert any("rank 1/2" in l for l in lines)
