"""A graphed two-rank training step with the BertAdam step inside the graph (skipped with fewer than two visible GPUs): four steps
of GraphedStep(model, sync, optimizer=...) must leave the parameters of the same four eager two-rank steps with the default
BertAdam after each, bit for bit (deterministic mode; the sum of two ranks has one order)."""
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
from visualbert_b200 import BertAdam, BertConfig, TrainVisualBERTObjective, graphs, synthetic
from visualbert_b200.parallel import FlatGradSync, shard_batch
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dev = torch.device("cuda", rank)
dist.init_process_group("nccl", device_id=dev)
torch.use_deterministic_algorithms(True)
cfg = synthetic.bert_config_dict(2, 128, 2, 256, vocab=512)


def replica():
    model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), "nlvr", visual_embedding_dim=64)
    model.load_state_dict(synthetic.init_state_dict(cfg, "nlvr", 64, seed=0), strict=False)
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    model.to(dev).train(True)
    model.bert.set_dropout_state({"seed": 9, "step": 100})
    opt = BertAdam([{"params": [p for n, p in model.named_parameters() if "bias" not in n], "weight_decay": 0.01},
                    {"params": [p for n, p in model.named_parameters() if "bias" in n], "weight_decay": 0.0}],
                   lr=1e-3, warmup=0.2, t_total=10, max_grad_norm=1.0)
    return model, FlatGradSync(model), opt


batches = []
for i in range(4):
    full = synthetic.make_batch(8, 20, 12, 64, head="nlvr", seed=5 + i, ragged=True, vocab=512)
    batches.append({k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in shard_batch(full, rank, world).items()})
ref, ref_sync, ref_opt = replica()
for b in batches:
    ref_sync.zero()
    loss = ref(**b)["loss"]
    (loss * ref_sync.loss_scale()).backward()
    ref_sync.allreduce(prescaled=True)
    ref_opt.step()
model, sync, opt = replica()
step = graphs.GraphedStep(model, sync, optimizer=opt)
for b in batches:
    step(b)
torch.cuda.synchronize()
assert len(step.graphs) == 1
diff = sum(int(not torch.equal(p.detach(), q.detach())) for p, q in zip(model.parameters(), ref.parameters()))
steps = sorted({s["step"] for s in opt.state_dict()["state"].values()})
print(f"RESULT rank {rank} differing {diff} steps {steps}")
dist.destroy_process_group()
'''


@two_gpus
def test_graphed_two_rank_step_with_optimizer_matches_eager(tmp_path):
    w = tmp_path / "worker.py"
    w.write_text(_WORKER)
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", CUBLAS_WORKSPACE_CONFIG=":4096:8")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", "29531", str(w), ROOT], capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    results = [x for x in r.stdout.splitlines() if x.startswith("RESULT")]
    assert len(results) == 2, r.stdout[-3000:]
    for line in results:
        assert line.split()[3:] == ["differing", "0", "steps", "[4]"], line
