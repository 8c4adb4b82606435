"""CPU-side checks of the deterministic-reduction switch (vb_set_deterministic, vb_deterministic_workspace_bytes): exported without
an ABI bump, declared in the header with the prototypes the binding uses, off by default, and a workspace formula that grows with
every dimension it is given (the pointers below are never dereferenced: no call here launches anything)."""
import ctypes
import os
import re

import pytest
import torch

from visualbert_b200 import _lib, ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_exported_and_declared_without_an_abi_bump():
    L = _lib.lib()
    names = {"vb_set_deterministic", "vb_deterministic_workspace_bytes"}
    assert names <= set(_lib.EXPORTS) and all(hasattr(L, n) for n in names)
    assert L.vb_abi_version() == _lib.ABI_VERSION == 4
    header = open(os.path.join(ROOT, "include", "vbert_b200.h")).read()
    assert re.search(r"int vb_set_deterministic\(void\* workspace, int64_t bytes\);", header)
    assert re.search(r"int64_t vb_deterministic_workspace_bytes\(int64_t rows, int32_t hidden, int32_t inter, int32_t vocab,\s*"
                     r"int32_t adam_chunks\);", header)
    assert L.vb_deterministic_workspace_bytes.restype is ctypes.c_int64


def test_switching_off_is_accepted_and_bad_workspaces_are_refused():
    L = _lib.lib()
    assert L.vb_set_deterministic(None, 0) == 0
    assert L.vb_set_deterministic(0x10000, 0) != 0 and "256-byte aligned" in L.vb_last_error().decode()
    assert L.vb_set_deterministic(0x10010, 1 << 20) != 0
    assert L.vb_set_deterministic(None, 0) == 0


def test_workspace_formula_is_monotone_and_aligned():
    L = _lib.lib()
    f = L.vb_deterministic_workspace_bytes
    base = dict(rows=256 * 164, hidden=768, inter=3072, vocab=30522, adam_chunks=0)

    def ws(**kw):
        a = dict(base, **kw)
        return f(a["rows"], a["hidden"], a["inter"], a["vocab"], a["adam_chunks"])

    b0 = ws()
    assert b0 > 0 and b0 % 256 == 0
    rows = [1, 64, 1000, 8192, 41984, 64 * 356, 100000]
    assert [ws(rows=r) for r in sorted(rows)] == sorted(ws(rows=r) for r in rows)
    hid = [64, 128, 256, 512, 768, 1024]
    assert [ws(hidden=h, inter=4 * h) for h in hid] == sorted(ws(hidden=h, inter=4 * h) for h in hid)
    voc = [0, 1000, 4096, 30522, 50000]
    assert [ws(vocab=v) for v in voc] == sorted(ws(vocab=v) for v in voc)
    # a BertAdam-only workspace: one fp32 partial per chunk
    assert f(0, 0, 0, 0, 716) >= 716 * 4
    assert ws(adam_chunks=10 ** 6) >= 4 * 10 ** 6
    # the split-K slabs of the FFN weight gradients at cfg2 (72 x 3 CTAs on 132 SMs) are covered
    assert b0 >= 3 * 3072 * 768 * 4


@pytest.mark.parametrize("bad", [dict(rows=-1), dict(hidden=-8), dict(hidden=100), dict(vocab=-1), dict(adam_chunks=-1)])
def test_workspace_formula_refuses_bad_shapes(bad):
    a = dict(rows=1024, hidden=768, inter=3072, vocab=30522, adam_chunks=0, **{})
    a.update(bad)
    L = _lib.lib()
    assert L.vb_deterministic_workspace_bytes(a["rows"], a["hidden"], a["inter"], a["vocab"], a["adam_chunks"]) == -1
    assert "vb_deterministic_workspace_bytes" in L.vb_last_error().decode()


def test_python_scope_is_a_no_op_when_torch_determinism_is_off(monkeypatch):
    """ops.deterministic calls nothing unless torch.use_deterministic_algorithms is on (the default host path is unchanged)."""
    calls = []
    real = _lib.lib()

    class Spy:
        def __getattr__(self, name):
            if name in ("vb_set_deterministic", "vb_deterministic_workspace_bytes"):
                calls.append(name)
            return getattr(real, name)

    monkeypatch.setattr(_lib, "lib", lambda: Spy())
    assert not torch.are_deterministic_algorithms_enabled()
    with ops.deterministic("cpu", 1024, 768, 3072):
        pass
    assert calls == []
