"""BertAdam's graph-capturable mode without a GPU: the vb_adam_group mirror and schedule kinds against the header, the schedules
the device evaluates (and the ones it refuses), the host-side checks of vb_bert_adam_step_sched / vb_bert_adam_sched_check, the
mode switch and checkpoint steps as ints, and GraphedStep refusing an optimizer it cannot capture."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_group_mirror_matches_the_c_struct(tmp_path):
    from visualbert_b200 import _lib, optimization
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "vbert_b200.h"\n'
                   'int main(){printf("%zu %zu %zu %d %d %d %d\\n", sizeof(vb_adam_group), offsetof(vb_adam_group, weight_decay),'
                   'offsetof(vb_adam_group, schedule), VB_SCHED_CONSTANT, VB_SCHED_WARMUP_CONSTANT, VB_SCHED_WARMUP_LINEAR,'
                   'VB_SCHED_WARMUP_COSINE);return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [ctypes.sizeof(_lib.AdamGroup), _lib.AdamGroup.weight_decay.offset, _lib.AdamGroup.schedule.offset,
                   _lib.VB_SCHED_CONSTANT, _lib.VB_SCHED_WARMUP_CONSTANT, _lib.VB_SCHED_WARMUP_LINEAR, _lib.VB_SCHED_WARMUP_COSINE]
    assert optimization._GROUP_DTYPE.itemsize == got[0]
    header = open(os.path.join(ROOT, "include", "vbert_b200.h")).read()
    assert int(re.search(r"#define VB_ABI_VERSION (\d+)", header).group(1)) == _lib.ABI_VERSION == _lib.lib().vb_abi_version()


def _params():
    return [torch.nn.Parameter(torch.zeros(4)), torch.nn.Parameter(torch.zeros(3))]


@pytest.mark.parametrize("name", ["none", "warmup_constant", "warmup_linear", "warmup_cosine"])
def test_capturable_mode_accepts_the_four_schedules(name):
    from visualbert_b200 import BertAdam
    opt = BertAdam(_params(), lr=1e-3, warmup=0.1, t_total=100, schedule=name)
    assert opt.set_graph_capturable(True) is opt and opt._capturable
    opt.set_graph_capturable(False)
    assert not opt._capturable


def test_capturable_mode_refuses_schedules_the_device_cannot_evaluate():
    from visualbert_b200 import BertAdam, optimization

    class Halved(optimization.WarmupLinearSchedule):
        def get_lr_(self, progress):
            return 0.5 * super().get_lr_(progress)

    class Custom(optimization._LRSchedule):
        pass

    for sched in (Halved(warmup=0.1, t_total=100), Custom(warmup=0.1, t_total=100), optimization._LRSchedule()):
        opt = BertAdam(_params(), lr=1e-3, schedule=sched)
        with pytest.raises(ValueError, match="SCHEDULES"):
            opt.set_graph_capturable(True)
        assert not opt._capturable
    opt = BertAdam(_params(), lr=1e-3, warmup=0.1, t_total=0)   # the host schedule divides by t_total
    with pytest.raises(ValueError, match="t_total"):
        opt.set_graph_capturable(True)
    # one bad group among good ones refuses the switch
    p = _params()
    opt = BertAdam([{"params": [p[0]]}, {"params": [p[1]], "schedule": Halved(warmup=0.1, t_total=10)}], lr=1e-3)
    with pytest.raises(ValueError, match="Halved"):
        opt.set_graph_capturable(True)


def _tab(groups_of_tensors, numel=40000):
    from visualbert_b200 import _lib, optimization
    tab = np.zeros(len(groups_of_tensors), dtype=optimization._TABLE_DTYPE)
    chunk = 0
    for i, g in enumerate(groups_of_tensors):
        tab[i] = (0x10000, 0x20000, 0x30000, 0x40000, numel, 0.0, 0.0, chunk, g)
        chunk += (numel + _lib.VB_ADAM_CHUNK - 1) // _lib.VB_ADAM_CHUNK
    return tab, chunk


def _groups(kinds):
    from visualbert_b200 import optimization
    return np.array([(1e-3, 0.1, 100.0, 0.5, 0.01, k) for k in kinds], dtype=optimization._GROUP_DTYPE)


def _ptr(a):
    return ctypes.c_void_p(a.ctypes.data)


def test_sched_step_checks_pointers_and_hyperparameters_before_any_cuda_call():
    from visualbert_b200 import _lib
    L = _lib.lib()
    D = ctypes.c_double
    P = ctypes.c_void_p
    rc = L.vb_bert_adam_step_sched(None, 2, 4, P(0x1000), 1, P(0x2000), P(0x3000), None, D(0.9), D(0.999), D(1e-6), D(1.0), None)
    assert rc != 0 and b"null table" in L.vb_last_error()
    rc = L.vb_bert_adam_step_sched(P(0x1000), 2, 4, None, 1, P(0x2000), P(0x3000), None, D(0.9), D(0.999), D(1e-6), D(1.0), None)
    assert rc != 0 and b"null table / groups" in L.vb_last_error()
    rc = L.vb_bert_adam_step_sched(P(0x1000), 2, 4, P(0x1000), 0, P(0x2000), P(0x3000), None, D(0.9), D(0.999), D(1e-6), D(1.0),
                                   None)
    assert rc != 0 and b"no groups" in L.vb_last_error()
    rc = L.vb_bert_adam_step_sched(P(0x1000), 2, 4, P(0x1000), 1, P(0x2000), P(0x3000), None, D(1.0), D(0.999), D(1e-6), D(1.0),
                                   None)
    assert rc != 0 and b"bad b1 / b2 / eps" in L.vb_last_error()


def test_sched_check_reports_bad_groups_and_layouts():
    from visualbert_b200 import _lib
    L = _lib.lib()
    tab, n_chunks = _tab([0, 1, 1])
    good = _groups([_lib.VB_SCHED_WARMUP_LINEAR, _lib.VB_SCHED_WARMUP_COSINE])
    assert L.vb_bert_adam_sched_check(_ptr(tab), 3, n_chunks, _ptr(good), 2) == 0
    assert L.vb_bert_adam_sched_check(None, 3, n_chunks, _ptr(good), 2) != 0
    assert b"null table" in L.vb_last_error()
    assert L.vb_bert_adam_sched_check(_ptr(tab), 3, n_chunks, _ptr(good), 1) != 0   # group 1 does not exist
    assert b"group index 1 out of range" in L.vb_last_error()
    bad, _ = _tab([0, -1, 1])
    assert L.vb_bert_adam_sched_check(_ptr(bad), 3, n_chunks, _ptr(good), 2) != 0
    assert b"group index -1 out of range" in L.vb_last_error()
    for kind in (4, -1):
        assert L.vb_bert_adam_sched_check(_ptr(tab), 3, n_chunks, _ptr(_groups([0, kind])), 2) != 0
        assert b"unknown schedule kind" in L.vb_last_error()
    g = good.copy()
    g["t_total"][1] = 0.0
    assert L.vb_bert_adam_sched_check(_ptr(tab), 3, n_chunks, _ptr(g), 2) != 0 and b"t_total 0" in L.vb_last_error()
    g = good.copy()
    g["warmup"][0] = 1.0
    assert L.vb_bert_adam_sched_check(_ptr(tab), 3, n_chunks, _ptr(g), 2) != 0 and b"warmup" in L.vb_last_error()
    assert L.vb_bert_adam_sched_check(_ptr(tab), 3, n_chunks + 1, _ptr(good), 2) != 0 and b"chunks" in L.vb_last_error()


def test_state_dict_steps_are_ints_and_load_takes_ints_or_tensors():
    from visualbert_b200 import BertAdam
    p = _params()
    opt = BertAdam(p, lr=1e-3, warmup=0.1, t_total=100)
    for i, q in enumerate(p):   # as a checkpoint of a step taken elsewhere would leave it
        opt.state[q].update(step=torch.tensor(5 + i), next_m=torch.zeros_like(q), next_v=torch.zeros_like(q))
    sd = opt.state_dict()
    assert [s["step"] for s in sd["state"].values()] == [5, 6]
    assert all(type(s["step"]) is int for s in sd["state"].values())
    assert torch.is_tensor(opt.state[p[0]]["step"])   # state_dict() leaves the live state alone
    opt2 = BertAdam(_params(), lr=1e-3, warmup=0.1, t_total=100)
    opt2.load_state_dict(sd)
    assert [opt2.state[q]["step"] for q in opt2.param_groups[0]["params"]] == [5, 6]
    opt3 = BertAdam(_params(), lr=1e-3, warmup=0.1, t_total=100)
    sd["state"][0]["step"] = torch.tensor(9)
    opt3.load_state_dict(sd)   # a tensor step in the default mode comes back as an int
    assert [type(opt3.state[q]["step"]) for q in opt3.param_groups[0]["params"]] == [int, int]
    assert opt3.state[opt3.param_groups[0]["params"][0]]["step"] == 9
    gen = opt3.plan_generation
    opt3.load_state_dict(sd)
    assert opt3.plan_generation > gen   # a graph captured before the load is stale


def test_graphed_step_refuses_other_optimizers_and_changes_nothing():
    from visualbert_b200 import BertConfig, TrainVisualBERTObjective, graphs, synthetic
    cfg = BertConfig.from_dict(synthetic.bert_config_dict(1, 128, 2, 256, vocab=64))
    model = TrainVisualBERTObjective(cfg, "nlvr", visual_embedding_dim=64).train(True)
    for opt in (torch.optim.SGD(model.parameters(), lr=0.1), torch.optim.Adam(model.parameters(), lr=0.1, capturable=True)):
        with pytest.raises(ValueError, match="BertAdam"):
            graphs.GraphedStep(model, sync=None, optimizer=opt)
    assert not model.bert._capturable
