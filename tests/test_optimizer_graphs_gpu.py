"""BertAdam in graph-capturable mode (vb_bert_adam_step_sched) on the GPU.

- The learning rate the kernels compute from the device step counters (lr_out) has the bits of the host's
  np.float32(lr * schedule.get_lr(step)) at every step, for every schedule kind (cosine: within one fp32 ulp).
- The eager step in this mode equals the default step bit for bit (parameters, moments, steps) over groups, clipping, multi-chunk
  and unaligned tensors and deterministic mode, and matches the reference golden.
- opt.step() captured in a CUDA graph and replayed equals eager steps; a group lr changed between replays applies from the next.
- graphs.GraphedStep(optimizer=...) equals eager steps with the default BertAdam after each; checkpoints round-trip to the default
  mode; load_state_dict evicts the graph; eval forwards see the updated weights; refusals leave nothing cached.
- The default step launches the kernels and grids it did before.
"""
import copy
import json
import os

import numpy as np
import pytest
import torch

import golden_util  # noqa: F401  (puts oracle/ on sys.path)
import adam_util

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLD = os.path.join(os.path.dirname(__file__), "golden", "bert_adam.npz")


@pytest.fixture(autouse=True)
def _cleanup():
    yield
    torch.use_deterministic_algorithms(False)
    from visualbert_b200 import _lib
    _lib.lib().vb_set_deterministic(None, 0)
    _lib.lib().vb_set_dropout_offset(None)


def _bits(x):
    return np.float32(x).view(np.uint32)


PAIRS = [(0.1, 100), (0.0, 100), (0.25, 37), (0.5, 250), (0.002, 1000), (0.1, -1)]


@pytest.mark.parametrize("name", ["none", "warmup_constant", "warmup_linear", "warmup_cosine"])
def test_device_schedule_equals_host_schedule(name):
    """One single-element parameter per (warmup, t_total) pair, each its own group with its own base lr; every step from 0 to
    t_total + 50 (the longest, 1050, for all)."""
    from visualbert_b200 import BertAdam, optimization
    params, groups = [], []
    for i, (warmup, t_total) in enumerate(PAIRS):
        p = torch.nn.Parameter(torch.zeros(1, device=DEV))
        p.grad = torch.zeros(1, device=DEV)
        params.append(p)
        groups.append({"params": [p], "lr": [1e-3, 5e-5, 0.1, 2e-4, 3.0, 1e-4][i],
                       "schedule": optimization.SCHEDULES[name](warmup=warmup, t_total=t_total)})
    opt = BertAdam(groups, lr=1.0, weight_decay=0.0).set_graph_capturable(True)
    n_steps = max(t for _, t in PAIRS) + 51
    differ = 0
    for step in range(n_steps):
        opt.step()
        got = opt.last_lr()
        for p, g in zip(params, groups):
            want = np.float32(g["lr"] * g["schedule"].get_lr(step))
            have = np.float32(got[p])
            if name == "warmup_cosine":
                d = abs(int(_bits(have).astype(np.int64)) - int(_bits(want).astype(np.int64)))
                assert d <= 1, (step, g["schedule"].warmup, g["schedule"].t_total, have, want)
                differ += d != 0
            else:
                assert _bits(have) == _bits(want), (step, g["schedule"].warmup, g["schedule"].t_total, have, want)
    assert all(int(opt.state[p]["step"]) == n_steps for p in params)
    if name == "warmup_cosine":
        print(f"warmup_cosine: {differ} of {n_steps * len(PAIRS)} learning rates differ by one fp32 ulp from the host's")


def _flat_params(numels, offset, seed):
    """Views of one flat buffer at `offset` (offset 1: every view is misaligned for 16-byte access, the scalar path)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    flat_p = torch.randn(sum(numels) + offset, device=DEV, generator=g) * 0.1
    params, off = [], offset
    for n in numels:
        params.append(torch.nn.Parameter(flat_p[off: off + n]))
        off += n
    return params


def _groups(params):
    return [{"params": params[:3], "weight_decay": 0.01}, {"params": params[3:], "weight_decay": 0.0}]


@pytest.mark.parametrize("max_grad_norm", [1.0, -1.0])
@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("offset", [0, 1])
def test_capturable_eager_step_equals_default_step(max_grad_norm, det, offset):
    from visualbert_b200 import BertAdam
    numels = [100003, 32768, 7, 70001, 5, 65536 * 2 + 3]
    runs = []
    torch.use_deterministic_algorithms(det)
    for capturable in (False, True):
        params = _flat_params(numels, offset, seed=11)
        opt = BertAdam(_groups(params), lr=2e-3, warmup=0.3, t_total=8, max_grad_norm=max_grad_norm)
        opt.set_graph_capturable(capturable)
        g = torch.Generator(device=DEV).manual_seed(5)
        for s in range(6):
            for p in params:
                p.grad = torch.randn(p.shape, device=DEV, generator=g) * (10.0 if s % 2 else 0.01)
            opt.step()
        runs.append((params, opt))
    (p0, o0), (p1, o1) = runs
    # outside deterministic mode the clip's norm of a multi-chunk tensor is a sum of float atomics, whose order varies from run
    # to run: there the two modes agree to rounding, elsewhere bit for bit
    exact = det or max_grad_norm <= 0
    for a, b in zip(p0, p1):
        for x, y in ((a.detach(), b.detach()), (o0.state[a]["next_m"], o1.state[b]["next_m"]),
                     (o0.state[a]["next_v"], o1.state[b]["next_v"])):
            if exact or x.numel() <= 32768:
                assert torch.equal(x, y)
            else:
                torch.testing.assert_close(x, y, rtol=1e-5, atol=1e-9)
        assert o0.state[a]["step"] == 6 and torch.is_tensor(o1.state[b]["step"]) and int(o1.state[b]["step"]) == 6
    assert o0.get_lr() == o1.get_lr()


def test_capturable_step_matches_reference_golden():
    """As test_optimizer_gpu.test_bert_adam_matches_reference_golden, in graph-capturable mode."""
    from visualbert_b200 import BertAdam
    gold = np.load(GOLD)
    init, grads = adam_util.scenario()
    params = [torch.nn.Parameter(t.clone().to(DEV)) for t in init]
    opt = BertAdam([{"params": params[:3], "weight_decay": 0.01}, {"params": params[3:], "weight_decay": 0.0}], **adam_util.HYPER)
    opt.set_graph_capturable(True)
    for s in range(adam_util.STEPS):
        for i, p in enumerate(params):
            p.grad = grads[s][i].clone().to(DEV)
        versions = [p._version for p in params]
        opt.step()
        assert all(p._version > v for p, v in zip(params, versions))
        for i, p in enumerate(params):
            assert int(opt.state[p]["step"]) == s + 1
            for name, t in (("p", p.detach()), ("m", opt.state[p]["next_m"]), ("v", opt.state[p]["next_v"])):
                np.testing.assert_allclose(t.cpu().numpy(), gold[f"{name}{i}_s{s}"], rtol=1e-5, atol=1e-8,
                                           err_msg=f"{name}{i} step {s}")
    assert all(type(s["step"]) is int and s["step"] == adam_util.STEPS for s in opt.state_dict()["state"].values())


@pytest.mark.parametrize("det", [False, True])
def test_captured_optimizer_step_replays_equal_eager_steps(det):
    """Clipping on in deterministic mode; off outside it, where a multi-chunk norm is a sum of float atomics in no fixed order."""
    from visualbert_b200 import BertAdam
    numels = [100003, 7, 70001, 5]
    torch.use_deterministic_algorithms(det)
    g = torch.Generator(device=DEV).manual_seed(3)
    grads = [[torch.randn(n, device=DEV, generator=g) for n in numels] for _ in range(7)]

    def make(capturable):
        params = _flat_params(numels, 1, seed=4)
        for p in params:
            p.grad = torch.zeros_like(p)
        opt = BertAdam([{"params": params[:2], "weight_decay": 0.01}, {"params": params[2:], "weight_decay": 0.0}],
                       lr=1e-3, warmup=0.2, t_total=10, max_grad_norm=1.0 if det else -1.0)
        return params, opt.set_graph_capturable(capturable)

    ref_p, ref_o = make(False)
    params, opt = make(True)
    for s in range(7):
        if s == 4:   # a new lr applies from the next step on
            ref_o.param_groups[1]["lr"] = 5e-3
        for p, gr in zip(ref_p, grads[s]):
            p.grad.copy_(gr)
        ref_o.step()
    # step 0 eagerly on a side stream (allocates the moments and tables), then capture one step and replay it six times
    for p, gr in zip(params, grads[0]):
        p.grad.copy_(gr)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        opt.step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        opt.step()
    assert all(int(opt.state[p]["step"]) == 1 for p in params)   # capture runs nothing
    for s in range(1, 7):
        if s == 4:
            opt.param_groups[1]["lr"] = 5e-3
            opt.sync_group_table()
        for p, gr in zip(params, grads[s]):
            p.grad.copy_(gr)
        graph.replay()
    for a, b in zip(ref_p, params):
        assert torch.equal(a.detach(), b.detach())
        assert torch.equal(ref_o.state[a]["next_m"], opt.state[b]["next_m"])
        assert torch.equal(ref_o.state[a]["next_v"], opt.state[b]["next_v"])
        assert int(opt.state[b]["step"]) == ref_o.state[a]["step"] == 7
    want = np.float32(5e-3 * ref_o.param_groups[1]["schedule"].get_lr(6))
    assert np.float32(opt.last_lr()[params[3]]) == want


def _model(head, T, V, B=4, seed=1234):
    from visualbert_b200 import BertConfig, TrainVisualBERTObjective, synthetic
    cfg = synthetic.bert_config_dict(2, 128, 2, 256, vocab=512)
    model = TrainVisualBERTObjective(BertConfig.from_dict(cfg), head, visual_embedding_dim=64)
    model.load_state_dict(synthetic.init_state_dict(cfg, head, 64, seed=0), strict=False)
    for m in model.modules():   # torch's own dropout draws from torch's generator, whose sequence under capture is not ours
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    return model.to(DEV).train(True)


def _batches(head, T, V, n=6):
    from visualbert_b200 import synthetic
    out = []
    for i in range(n):
        b = synthetic.make_batch(4, T, V, 64, head=head, seed=100 + i, vocab=512, ragged=True)
        out.append({k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in b.items()})
    return out


def _opt(model, **kw):
    from visualbert_b200 import BertAdam
    named = list(model.named_parameters())
    nd = ("bias", "LayerNorm.bias", "LayerNorm.weight")
    return BertAdam([{"params": [p for n, p in named if not any(x in n for x in nd)], "weight_decay": 0.01},
                     {"params": [p for n, p in named if any(x in n for x in nd)], "weight_decay": 0.0}],
                    lr=1e-3, warmup=0.1, t_total=10, max_grad_norm=1.0, **kw)


def _eager(model, sync, opt, batches):
    losses = []
    for b in batches:
        sync.zero()
        out = model(**b)
        out["loss"].backward()
        losses.append(out["loss"].detach().clone())
        opt.step()
    return losses


def _same(a, b):
    assert len(a) == len(b)
    for i, (u, v) in enumerate(zip(a, b)):
        assert torch.equal(u, v), i


STATE = {"seed": 77, "step": 2 ** 32 - 3}


@pytest.mark.parametrize("head,T,V", [("nlvr", 40, 36), ("vqa", 20, 36)])
def test_graphed_step_with_optimizer_equals_eager_steps(head, T, V, monkeypatch):
    from visualbert_b200 import graphs, parallel
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    torch.use_deterministic_algorithms(True)
    batches = _batches(head, T, V)
    ref = _model(head, T, V)
    ref.bert.set_dropout_state(STATE)
    ref_sync = parallel.FlatGradSync(ref)
    ref_opt = _opt(ref)
    ref_losses = _eager(ref, ref_sync, ref_opt, batches)

    model = _model(head, T, V)
    model.bert.set_dropout_state(STATE)
    sync = parallel.FlatGradSync(model)
    opt = _opt(model)
    step = graphs.GraphedStep(model, sync, optimizer=opt)
    losses = [step(b)["loss"].detach().clone() for b in batches]
    assert len(step.graphs) == 1
    _same(losses, ref_losses)
    _same([p.detach() for p in model.parameters()], [p.detach() for p in ref.parameters()])
    _same([opt.state[p]["next_m"] for p in model.parameters()], [ref_opt.state[p]["next_m"] for p in ref.parameters()])
    assert model.bert.dropout_state() == ref.bert.dropout_state()
    steps = [s["step"] for s in opt.state_dict()["state"].values()]
    assert steps and all(type(s) is int and s == 6 for s in steps)


def test_checkpoint_round_trip_and_reload_evicts_the_graph(monkeypatch):
    from visualbert_b200 import BertAdam, graphs, parallel
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    torch.use_deterministic_algorithms(True)
    batches = _batches("nlvr", 24, 16)
    ref = _model("nlvr", 24, 16)
    ref.bert.set_dropout_state(STATE)
    ref_sync = parallel.FlatGradSync(ref)
    _eager(ref, ref_sync, _opt(ref), batches)

    model = _model("nlvr", 24, 16)
    model.bert.set_dropout_state(STATE)
    sync = parallel.FlatGradSync(model)
    opt = _opt(model)
    step = graphs.GraphedStep(model, sync, optimizer=opt)
    for b in batches[:3]:
        step(b)
    ckpt = copy.deepcopy(opt.state_dict())
    weights = copy.deepcopy(model.state_dict())
    dstate = model.bert.dropout_state()
    assert all(type(s["step"]) is int and s["step"] == 3 for s in ckpt["state"].values())

    # a default-mode BertAdam on a fresh model continues from the checkpoint
    fresh = _model("nlvr", 24, 16)
    fresh.load_state_dict(weights)
    fresh.bert.set_dropout_state(dstate)
    fresh_sync = parallel.FlatGradSync(fresh)
    fresh_opt = _opt(fresh)
    fresh_opt.load_state_dict(copy.deepcopy(ckpt))
    assert isinstance(fresh_opt, BertAdam) and not fresh_opt._capturable
    _eager(fresh, fresh_sync, fresh_opt, batches[3:])
    _same([p.detach() for p in fresh.parameters()], [p.detach() for p in ref.parameters()])

    # the captured optimizer reloads the same checkpoint: its tables are rebuilt, so the graph is captured again
    opt.load_state_dict(copy.deepcopy(ckpt))
    for b in batches[3:]:
        step(b)
    assert len(step.graphs) == 1
    _same([p.detach() for p in model.parameters()], [p.detach() for p in ref.parameters()])
    assert all(s["step"] == 6 for s in opt.state_dict()["state"].values())


def test_eval_forward_after_graphed_steps_sees_the_updated_weights():
    from visualbert_b200 import graphs, parallel
    batches = _batches("nlvr", 20, 12, n=4)
    model = _model("nlvr", 20, 12)
    sync = parallel.FlatGradSync(model)
    opt = _opt(model)
    step = graphs.GraphedStep(model, sync, optimizer=opt)
    with torch.no_grad():
        model.eval()
        model(**batches[0])   # fills the eval-mode bf16 weight cache with the initial weights
        model.train(True)
    for b in batches:
        step(b)
    model.bert.set_graph_capturable(False)
    opt.set_graph_capturable(False)
    model.eval()
    twin = _model("nlvr", 20, 12).eval()
    twin.load_state_dict(model.state_dict())
    with torch.no_grad():
        assert torch.equal(model(**batches[0])["logits"], twin(**batches[0])["logits"])
    assert all(type(s["step"]) is int for s in (opt.state[p] for p in model.parameters() if p in opt.state))


def test_refusals_leave_nothing_cached():
    from visualbert_b200 import graphs, parallel
    batch = _batches("nlvr", 20, 12, n=1)[0]
    model = _model("nlvr", 20, 12)
    sync = parallel.FlatGradSync(model)
    with pytest.raises(ValueError, match="BertAdam"):
        graphs.GraphedStep(model, sync, optimizer=torch.optim.SGD(model.parameters(), lr=0.1))
    assert not model.bert._capturable
    # capture before any eager step of the optimizer: its moments would be allocated (and zeroed) inside the graph
    opt = _opt(model)
    step = graphs.GraphedStep(model, sync, optimizer=opt, warmup=0)
    sync.zero()
    model(**batch)["loss"].backward()   # the model's own workspaces are warm: the refusal is the optimizer's
    torch.cuda.synchronize()
    with pytest.raises(ValueError, match="next_m"):
        step(batch)
    assert len(step.graphs) == 0 and all(len(s) == 0 for s in opt.state.values()) and not opt._plans
    torch.cuda.synchronize()
    # an optimizer switched back to the default mode is refused at capture, after its eager warm-up step ran
    step = graphs.GraphedStep(model, sync, optimizer=opt)
    opt.set_graph_capturable(False)
    step(batch)
    with pytest.raises(ValueError, match="graph-capturable"):
        step(batch)
    assert len(step.graphs) == 0
    torch.cuda.synchronize()


_PROFILE = r"""
import json, sys, torch
sys.path.insert(0, sys.argv[1])
from torch.profiler import ProfilerActivity, profile
from visualbert_b200 import BertAdam, _lib
dev = "cuda:0"
flat = torch.randn(100003 + 7 + 70001, device=dev) * 0.1
params = [torch.nn.Parameter(flat[:100003]), torch.nn.Parameter(flat[100003:100010]), torch.nn.Parameter(flat[100010:])]
for p in params:
    p.grad = torch.randn_like(p)
opt = BertAdam(params, lr=1e-3, warmup=0.1, t_total=10)


def kernels(tag):
    opt.step()   # warm-up: tables built, modules loaded
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        opt.step()
        torch.cuda.synchronize()
    path = sys.argv[2] + "/" + tag + ".json"
    prof.export_chrome_trace(path)
    ev = json.load(open(path))["traceEvents"]
    return [(e["name"].split("(")[0], e["args"]["grid"], e["args"]["block"]) for e in ev
            if e.get("cat") == "kernel" and "adam" in e["name"]]


out = {"default": kernels("default")}
opt.set_graph_capturable(True)
out["sched"] = kernels("sched")
opt.set_graph_capturable(False)
out["default_again"] = kernels("default_again")
print("KERNELS " + json.dumps(out))
"""


def test_default_step_launches_the_same_kernels_and_grids(tmp_path):
    """Profiled in a process of its own: the kernel names and grids of one step in each mode."""
    import subprocess
    import sys
    from visualbert_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = tmp_path / "profile_adam.py"
    script.write_text(_PROFILE)
    r = subprocess.run([sys.executable, str(script), root, str(tmp_path)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    got = json.loads([x for x in r.stdout.splitlines() if x.startswith("KERNELS ")][0][len("KERNELS "):])
    n_chunks = sum((n + _lib.VB_ADAM_CHUNK - 1) // _lib.VB_ADAM_CHUNK for n in (100003, 7, 70001))
    default = [["vb::adam_sumsq_kernel", [n_chunks, 1, 1], [256, 1, 1]], ["vb::adam_update_kernel", [n_chunks, 1, 1], [256, 1, 1]]]
    assert got["default"] == default, got
    assert got["sched"] == [["vb::adam_sumsq_kernel", [n_chunks, 1, 1], [256, 1, 1]],
                            ["vb::adam_update_sched_kernel", [n_chunks, 1, 1], [256, 1, 1]],
                            ["vb::adam_step_advance_kernel", [1, 1, 1], [256, 1, 1]]], got
    assert got["default_again"] == default, got
