"""Single-image sequence parallelism over NVLink peer memory (SURVEY.md 8f-2) -- needs >= 2 H100s on one node.

Launches tests/sp_worker.py with one process per GPU (NCCL only for set-up and the final gather) and checks its report:
  * cudaIpc peer buffers, peer stores and the phase barrier work, and a barrier a peer never joins reports a time-out
    instead of hanging the GPU;
  * Flux.forward and the Euler sampler in sequence-parallel mode agree with the single-GPU path of the same library
    (only the attention key order differs: rel-L2 <= 1e-2 after a forward, <= 3e-2 after a trajectory) and stay inside
    the oracle / reference-golden tolerances of test_flux_gpu.py.
"""
import json
import os
import subprocess
import sys

import pytest
import torch

from conftest import REPO

pytestmark = pytest.mark.gpu


def _run(world, tmp_path, mode):
    out = tmp_path / "sp_report.json"
    port = 29500 + (os.getpid() % 500)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(REPO, "tests", "sp_worker.py"), str(out), mode]
    p = subprocess.run(cmd, cwd=REPO, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + "\n" + p.stderr[-3000:]
    return json.loads(out.read_text())


@pytest.mark.parametrize("world", [2, 4])
def test_sequence_parallel(tmp_path, world):
    if not torch.cuda.is_available() or torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs on one node")
    rep = _run(world, tmp_path, os.environ.get("VCB_SP_TEST_MODE", "quick"))
    assert rep["peer_store_ok"] and rep["barrier2_ok"] and rep["timeout_reported"]
    assert rep["small_ranks_identical"]
    assert rep["small_sp_vs_single"] < 1e-2, rep
    assert rep["small_sp_vs_oracle"] < 2e-2, rep
    assert rep["traj_shape_ok"] and rep["traj_x0_exact"]
    assert rep["traj_sp_vs_single"] < 3e-2, rep
    if rep["small_sp_vs_golden"] is not None:          # 2 ranks: the reference-generated 2-head fixtures apply
        assert rep["small_sp_vs_golden"] < 2.5e-2 and rep["traj_sp_vs_golden"] < 5e-2, rep
    if "big_sp_vs_single" in rep:
        assert rep["big_sp_vs_single"] < 1e-2, rep
