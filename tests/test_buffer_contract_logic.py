"""CPU tests of the buffer-contract harness (tests/_buffer_contract.py) on host tensors: a write one element past either end
of a framed buffer is reported with its offset, an in-bounds write is not, the body holds the poison, the body keeps the
allocation's alignment, and the torch stand-in forwards everything it does not frame."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _buffer_contract as BC  # noqa: E402


@pytest.mark.parametrize("dtype", [torch.uint8, torch.int32, torch.float32, torch.float64])
@pytest.mark.parametrize("shape", [(1,), (7,), (3, 5), (2, 3, 3)])
@pytest.mark.parametrize("side", ["left", "right"])
def test_writes_one_element_past_either_end_are_reported(dtype, shape, side):
    fr = BC.Framer(devices=("cpu",))
    t = fr.framed(shape, dtype, "cpu", 0xFF, name="t")
    es = t.element_size()
    flat = t.view(-1)
    store = torch.as_strided(flat, (flat.numel() + 2,), (1,), flat.storage_offset() - 1)   # one element each side
    assert fr.frames_intact() == []
    store[0 if side == "left" else -1] = 1
    bad = fr.frames_intact()
    assert len(bad) == 1 and bad[0][:2] == ("t", side)
    if side == "right":
        assert bad[0][2] == t.numel() * es                  # the first byte past the end
    else:
        assert -es <= bad[0][2] < 0                         # within the element just before the start


def test_in_bounds_writes_are_not_reported():
    fr = BC.Framer(devices=("cpu",))
    t = fr.framed((5, 3), torch.float32, "cpu", 0xFF, name="t")
    t[0, 0] = 1.0
    t[-1, -1] = -2.0
    t.fill_(0.5)
    assert fr.frames_intact() == []


@pytest.mark.parametrize("poison", BC.POISONS)
@pytest.mark.parametrize("dtype", [torch.uint8, torch.int16, torch.int32, torch.int64, torch.float32, torch.float64, torch.bfloat16])
def test_body_holds_the_poison_and_frames_the_canary(poison, dtype):
    fr = BC.Framer(devices=("cpu",))
    t = fr.framed((3, 7), dtype, "cpu", poison)
    assert t.is_contiguous() and t.shape == (3, 7) and t.dtype == dtype
    assert (t.contiguous().view(-1).view(torch.uint8) == poison).all()
    if poison == 0xFF and dtype.is_floating_point:
        assert torch.isnan(t).all()
    if poison == 0xFF and not dtype.is_floating_point and dtype != torch.uint8:
        assert (t == -1).all()
    raw = fr.bufs[-1][1].numpy()
    n = t.numel() * t.element_size()
    assert len(raw) == 2 * BC.FRAME + n and t.data_ptr() == fr.bufs[-1][1].data_ptr() + BC.FRAME
    assert (raw[:BC.FRAME] == BC.CANARY).all() and (raw[BC.FRAME + n:] == BC.CANARY).all()


def _align(p):
    return p & -p


@pytest.mark.parametrize("n", [1, 3, 4096, 4097])
def test_body_alignment_is_at_least_the_bases(n):
    fr = BC.Framer(devices=("cpu",))
    t = fr.framed((n,), torch.uint8, "cpu", 0)
    base = fr.bufs[-1][1].data_ptr()
    assert t.data_ptr() == base + BC.FRAME
    assert _align(t.data_ptr()) >= min(_align(base), BC.FRAME)


def test_poison_refills_the_body_only():
    fr = BC.Framer(devices=("cpu",))
    t = fr.framed((9,), torch.int32, "cpu", 0x00)
    fr.poison(t, 0xFF)
    assert (t == -1).all() and fr.frames_intact() == []
    with pytest.raises(KeyError):
        fr.poison(torch.zeros(3), 0)


def test_shim_frames_its_devices_and_forwards_everything_else():
    fr = BC.Framer(devices=("cpu",))
    shim = BC.TorchShim(fr, 0xFF)
    a = shim.empty(2, 3, device="cpu", dtype=torch.float32)
    b = shim.empty((4,), device=torch.device("cpu"), dtype=torch.int32)
    c = shim.empty_like(a)
    z = shim.zeros(5, device="cpu", dtype=torch.uint8)
    e = shim.empty(torch.Size([2, 2]), device="cpu", dtype=torch.uint8)
    assert len(fr.bufs) == 5
    assert torch.isnan(a).all() and (b == -1).all() and torch.isnan(c).all() and (z == 0).all() and (e == 255).all()
    assert c.shape == a.shape and c.dtype == a.dtype and e.shape == (2, 2)
    host = shim.empty(6, dtype=torch.uint8)                  # no device: a host allocation passes through
    assert len(fr.bufs) == 5 and host.shape == (6,)
    assert shim.float32 is torch.float32 and shim.Tensor is torch.Tensor and shim.from_numpy is torch.from_numpy
    assert shim.cuda is torch.cuda and shim.device is torch.device
    assert isinstance(a, shim.Tensor)
    gpu_shim = BC.TorchShim(BC.Framer(), 0xFF)               # the default framer frames CUDA only
    plain = gpu_shim.empty(3, device="cpu", dtype=torch.float32)
    assert gpu_shim._framer.bufs == [] and plain.shape == (3,)


def test_under_both_poisons_catches_a_stale_read_and_a_frame_write(monkeypatch):
    import types
    fake_ops = types.SimpleNamespace(torch=torch)

    def run(monkeypatch, body):
        res = []
        for poison in BC.POISONS:
            fr = BC.Framer(devices=("cpu",))
            with monkeypatch.context() as mp:
                mp.setattr(fake_ops, "torch", BC.TorchShim(fr, poison))
                res.append((BC.to_host(body(fake_ops)), fr.frames_intact()))
        return res

    def good(o):
        out = o.torch.empty(4, device="cpu", dtype=torch.float32)
        out.fill_(2.0)
        return out

    def stale(o):                                           # leaves the last element unwritten
        out = o.torch.empty(4, device="cpu", dtype=torch.float32)
        out[:3] = 2.0
        return out

    def over(o):                                            # writes one element past the end
        out = o.torch.empty(4, device="cpu", dtype=torch.float32)
        torch.as_strided(out, (5,), (1,)).fill_(2.0)
        return out

    (r0, f0), (r1, f1) = run(monkeypatch, good)
    BC.bit_equal(r0, r1)
    assert f0 == f1 == []
    (r0, _), (r1, _) = run(monkeypatch, stale)
    with pytest.raises(AssertionError):
        BC.bit_equal(r0, r1)
    (_, f0), (_, f1) = run(monkeypatch, over)
    assert f0 == f1 == [("empty[4]", "right", 16)]
