"""Image-wise data-parallel infer on 2 GPUs (torchrun): the gathered dict must equal the single-GPU dict bit for bit
(no cross-image op on the path), with the default peer-memory gather (copy-engine pulls over CUDA-IPC buffers, outputs
written straight into the send slot) and with the NCCL fallback.  Skipped with fewer than 2 GPUs."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = r"""
import copy, json, os, sys
sys.path[:0] = [sys.argv[1], os.path.join(sys.argv[1], "oracle")]
import torch, torch.distributed as dist
from unidepth_b200 import UniDepthV2
from unidepth_b200 import parallel
from unidepth_b200.parallel import infer_sharded, shard_bounds
from unidepth_b200.synthetic import synthetic_state_dict
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
dev = torch.device("cuda", int(os.environ["LOCAL_RANK"]))
dist.init_process_group("nccl", device_id=dev)
cfg = json.load(open(os.path.join(sys.argv[1], "tests", "golden", "config_v2_vitl14.json")))
cfg["model"]["pixel_encoder"]["arch_override"] = {"depth": 4}
cfg["model"]["pixel_encoder"]["output_idx"] = [1, 2, 3, 4]
m = UniDepthV2(copy.deepcopy(cfg))
m.load_state_dict(synthetic_state_dict(cfg, 0, device=dev), strict=True)
m = m.to(dev).eval()
g = torch.Generator().manual_seed(7)
rgb = torch.randint(0, 256, (4, 3, 240, 320), dtype=torch.uint8, generator=g)
import warnings; warnings.simplefilter("ignore")
def same(got, tag):
    bad = [k for k in single if not torch.equal(got[k].float(), single[k].float())]
    if bad:
        k = bad[0]
        d = (got[k].float() - single[k].float()).abs()
        print(f"rank {rank}: MISMATCH in {tag}: keys {bad}; {k}: max abs diff {d.max().item():.3e}, "
              f"per-image max {[round(x, 6) for x in d.flatten(1).max(1).values.tolist()]}", flush=True)
    return not bad

# order matters: the FIRST call of the model captures the small (B=2) graph, then a gather, then the larger (B=4) graph --
# the sequence that exposed the use-after-free of the ray-frequency table (unidepthv2.py::_run)
full = infer_sharded(m, rgb)
single = m.infer(rgb)
ok = same(full, "first synchronous gather")
# pipelined form: three gathers in flight one after the other, replays of the older (B=2) graph after the
# capture of the larger (B=4) one
pend = [infer_sharded(m, rgb, async_op=True) for _ in range(3)]
for i, p in enumerate(pend):
    ok &= same(p.wait(), f"pipelined gather {i}")
# outputs produced straight into the send slot (model.output_buffers = the slot's views): no staging copy
lo, hi = shard_bounds(4, rank, world)
loc = m.infer(rgb[lo:hi])
in_slot = 0
for _ in range(3):
    m.output_buffers = parallel.output_views(loc)
    in_slot += m.output_buffers is not None
    ok &= same(infer_sharded(m, rgb), "gather of outputs written in place")
m.output_buffers = None
mode = parallel.gather_mode()
if mode == "p2p":
    setup_ok = parallel._p2p_failed[0] is None and len(parallel._p2p_cache) > 0 and in_slot == 3
    no_timeout = all(not pg.timed_out() for pg in parallel._p2p_cache.values())
    print(f"rank {rank}: p2p set up {setup_ok} (in-slot steps {in_slot}), no barrier timeout {no_timeout}", flush=True)
    ok &= setup_ok and no_timeout
print(f"rank {rank}: mode {mode} (p2p objects {len(parallel._p2p_cache)}, failure {parallel._p2p_failed[0]}), "
      f"gathered == single-GPU: {ok}", flush=True)
dist.destroy_process_group()
sys.exit(0 if ok else 1)
"""


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
def test_two_gpu_gather_equals_single_gpu(tmp_path, mode):
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29611" if mode == "p2p" else "29612", str(script), ROOT]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env={**os.environ, "UDB_GATHER": mode})
    print(out.stdout[-2000:], out.stderr[-2000:])
    assert out.returncode == 0
