"""A graphed training step across two ranks (skipped with fewer than two visible GPUs): GraphedStep captures the NCCL all-reduce
of FlatGradSync together with the step, and its flat gradients must equal those of the eager two-rank step at the same dropout
state (deterministic mode, so both ranks' gradients are reproducible; the sum of two ranks has one order)."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
two_gpus = pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs 2 GPUs")

_WORKER = r'''
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from visualbert_b200 import BertConfig, TrainVisualBERTObjective, graphs, synthetic
from visualbert_b200.parallel import FlatGradSync, shard_batch
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dev = torch.device("cuda", rank)
dist.init_process_group("nccl", device_id=dev)
torch.use_deterministic_algorithms(True)
cfg = synthetic.bert_config_dict(2, 128, 2, 256, vocab=512)
model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), "nlvr", visual_embedding_dim=64)
model.load_state_dict(synthetic.init_state_dict(cfg, "nlvr", 64, seed=0), strict=False)
for m in model.modules():
    if isinstance(m, torch.nn.Dropout):
        m.p = 0.0
model.to(dev).train(True)
full = synthetic.make_batch(8, 20, 12, 64, head="nlvr", seed=5, ragged=True, vocab=512)
mine = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in shard_batch(full, rank, world).items()}
sync = FlatGradSync(model)
state = {"seed": 9, "step": 100}
# eager two-rank step
model.bert.set_dropout_state(state)
sync.zero()
loss = model(**mine)["loss"]
(loss * sync.loss_scale()).backward()
ref = sync.allreduce(prescaled=True).clone()
# graphed: eager warm-up, then capture + replay (all-reduce inside the graph), each at the same dropout state
step = graphs.GraphedStep(model, sync)
errs = []
for _ in range(3):
    model.bert.set_dropout_state(state)
    step(mine)
    torch.cuda.synchronize()
    errs.append(((sync.flat - ref).norm() / ref.norm()).item())
assert len(step.graphs) == 1
if rank == 0:
    print("RESULT " + " ".join(f"{e:.3e}" for e in errs))
dist.destroy_process_group()
'''


@two_gpus
def test_graphed_two_rank_step_matches_eager(tmp_path):
    w = tmp_path / "worker.py"
    w.write_text(_WORKER)
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", CUBLAS_WORKSPACE_CONFIG=":4096:8")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", "29527", str(w), ROOT], capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    errs = [float(x) for x in [x for x in r.stdout.splitlines() if x.startswith("RESULT")][0].split()[1:]]
    assert all(e == 0.0 for e in errs), errs
