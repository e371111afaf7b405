"""CPU: the (head_dim, group) layouts the engine can run.  The attention kernel puts all group x M
query rows of a kv head on one CTA, and the engine never launches fewer than 16 tokens in the prompt
pass (engine.cu: prompt_attn_rows) while a verify block carries up to 16: a layout whose 16-token
launch does not fit the 227 KiB of shared memory cannot run, and `lsk_create` refuses it before any
CUDA call.  `lsk_plan_attention` reports ok = 0 for the same layouts at every m.

The largest group per head_dim follows from attention.cuh's attn_smem_plan at 16 tokens and 2 ring
stages: 128 header + 2 x 64-key K/V stages + the merge buffer + 16 x group partial rows of
(head_dim + 2) floats."""
import ctypes as C

import pytest

from layerskip_b200 import _lib
from layerskip_b200.weights import LlamaArch

SMS = 132
LARGEST_GROUP = {128: 16, 64: 43, 32: 95}      # 232 064 / 231 424 / 231 936 of 232 448 bytes


def _create(head_dim, n_heads, n_kv_heads, n_layers):
    """lsk_create's return code and error.  n_layers = 0 fails the LAST argument check, so an
    accepted layout reaches "bad n_layers" without touching the device."""
    lib = _lib.load()
    cfg = _lib.lsk_config(vocab=512, hidden=256, inter=688, n_layers=n_layers, n_heads=n_heads,
                          n_kv_heads=n_kv_heads, head_dim=head_dim, rms_eps=1e-5, rope_theta=1e4,
                          max_ctx=256, tp_rank=0, tp_size=1)
    h = C.c_void_p()
    code = lib.lsk_create(C.byref(cfg), C.byref(h))
    assert not h.value, "lsk_create returned an engine for an invalid config"
    return code, lib.lsk_last_error().decode()


def _layout_accepted(head_dim, n_heads, n_kv_heads):
    code, err = _create(head_dim, n_heads, n_kv_heads, n_layers=0)
    assert code == -1, (code, err)
    if "bad n_layers" in err:
        return True
    assert "shared memory for a 16-token launch" in err, err
    return False


def _plan_ok(head_dim, n_heads, n_kv_heads, m):
    out = _lib.lsk_attn_plan()
    _lib.check(_lib.load().lsk_plan_attention(head_dim, n_heads, n_kv_heads, m, SMS, C.byref(out)))
    return out.ok == 1


def test_group_32_at_head_dim_128_is_refused_by_name():
    code, err = _create(128, 32, 1, n_layers=2)
    assert code == -1
    assert "group 32" in err and "head_dim 128" in err and "32 heads over 1 kv heads" in err, err
    for m in (1, 8, 9, 16, 128):
        assert not _plan_ok(128, 32, 1, m), m


@pytest.mark.parametrize("head_dim,n_heads,n_kv", [(128, 32, 2), (128, 16, 1), (64, 32, 1), (64, 43, 1),
                                                    (32, 95, 1), (128, 24, 8)])
def test_largest_fitting_groups_are_accepted(head_dim, n_heads, n_kv):
    assert _layout_accepted(head_dim, n_heads, n_kv)
    assert _plan_ok(head_dim, n_heads, n_kv, 16)
    out = _lib.lsk_attn_plan()
    _lib.check(_lib.load().lsk_plan_attention(head_dim, n_heads, n_kv, 16, SMS, C.byref(out)))
    assert out.smem_bytes <= out.smem_limit == 227 * 1024


def test_planner_and_create_agree_on_every_layout():
    for head_dim, largest in LARGEST_GROUP.items():
        for group in range(1, 2 * largest + 3):
            for n_kv in (1, 2, 8):
                accepted = _layout_accepted(head_dim, group * n_kv, n_kv)
                assert accepted == (group <= largest), (head_dim, group, n_kv)
                # a refused layout has no m the planner accepts; an accepted one runs 1 .. 16 rows
                for m in (1, 7, 16):
                    assert _plan_ok(head_dim, group * n_kv, n_kv, m) == accepted, (head_dim, group, n_kv, m)


def test_engine_raises_before_it_allocates(monkeypatch):
    """`Engine` reaches lsk_create with no allocation of its own and raises its refusal (the CUDA
    queries the constructor makes first are stubbed: this machine may have no device)."""
    import contextlib

    import torch

    from layerskip_b200.engine import Engine
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a: (_ for _ in ()).throw(RuntimeError("no query")))
    monkeypatch.setattr(torch.cuda, "get_device_properties",
                        lambda *a: type("Props", (), dict(multi_processor_count=132))())
    monkeypatch.setattr(torch.cuda, "device", lambda *a: contextlib.nullcontext())
    arch = LlamaArch(512, 4096, 11008, 2, 32, 1, 128)
    with pytest.raises(_lib.LskError, match="group 32"):
        Engine(arch, max_ctx=256, device="cuda:0", prefill_tc=False)


def test_batched_attention_entry_refuses_bad_shapes_before_the_device():
    """`lsk_test_attn_seqs` checks its shape on the host: more than 16 rows, a sequence shorter than
    its rows or longer than its slot, a slot that is not whole pages, splits outside [1, 8], a page
    map that is not a permutation.  Without a GPU an accepted shape fails only at the device."""
    import torch
    lib = _lib.load()
    dev = C.c_void_p(16)                                       # never dereferenced on a refusal

    def call(n_heads=8, n_kv=2, hd=128, rows=4, ctx=(4, 300, 640), slot=640, splits=4, perm=None):
        c = (C.c_int32 * len(ctx))(*ctx)
        p = None if perm is None else (C.c_int32 * len(perm))(*perm)
        return lib.lsk_test_attn_seqs(dev, dev, dev, n_heads, n_kv, hd, len(ctx), rows, c, slot, splits, p, dev)

    pages = 3 * 10
    for bad in (dict(rows=6), dict(ctx=(5,) * 17, rows=1), dict(ctx=(3, 300, 640)), dict(ctx=(4, 300, 641)),
                dict(slot=600, ctx=(4, 300, 600)), dict(slot=0, ctx=(0, 0, 0), rows=0), dict(splits=0),
                dict(splits=9), dict(hd=96), dict(n_heads=7), dict(perm=[0] * pages),
                dict(perm=list(range(1, pages + 1)))):
        assert call(**bad) == -1, bad                          # LSK_ERR_INVALID
    if not torch.cuda.is_available():
        assert call() == -2                                    # LSK_ERR_CUDA: the shape was accepted
        assert call(perm=list(reversed(range(pages)))) == -2
