"""The buffer contract every libudh entry point keeps: a kernel writes only its outputs, reads only its inputs, and its result
does not depend on what a workspace or output held before the call.

A framed buffer is one allocation with FRAME bytes on each side of the tensor a caller sees.  The frames hold a known byte
(CANARY for workspaces and outputs, the run's poison around inputs) and the body starts as the run's poison: 0xFF (NaN in
fp32, fp64 and bf16, -1 in the integer types, 255 in uint8) or 0x00.  FRAME = 4096 keeps the body at the allocator's own
alignment or better, so 16-byte vector access and TMA base alignment hold as they do without frames.

TorchShim stands in for `torch` inside `ops` (monkeypatch.setattr(ops, "torch", shim)): every CUDA torch.empty /
empty_like / zeros it serves is framed, the first two filled with the poison, and recorded so the frames can be checked after
torch.cuda.synchronize().  Host allocations (the pinned plans, the ctypes tables) pass through.  The host-built tables ops
copies with torch.from_numpy(...).to(dev) (tile lists, pair lists, ROI tables) are not framed."""
import numpy as np
import torch

FRAME = 4096
CANARY = 0x5A
POISONS = (0xFF, 0x00)


class Framer(object):
    """Allocates framed buffers and remembers them: frames_intact() lists every frame whose bytes changed."""

    def __init__(self, devices=("cuda",)):
        self.devices = tuple(devices)
        self.bufs = []                      # (name, raw uint8, body bytes, frame byte)

    def framed(self, shape, dtype, device, body, canary=CANARY, name=None):
        """-> a contiguous tensor of `shape` and `dtype`, the body filled with the byte `body`, inside one allocation whose
        FRAME bytes on each side hold the byte `canary`."""
        shape = tuple(int(s) for s in shape)
        nbytes = int(np.prod(shape, dtype=np.int64)) * torch.empty(0, dtype=dtype).element_size()
        raw = torch.empty(2 * FRAME + nbytes, dtype=torch.uint8, device=device)
        raw[:FRAME].fill_(canary)
        raw[FRAME + nbytes:].fill_(canary)
        raw[FRAME:FRAME + nbytes].fill_(body)
        self.bufs.append((name or "buf%d%s" % (len(self.bufs), list(shape)), raw, nbytes, canary))
        return raw[FRAME:FRAME + nbytes].view(dtype).view(shape)

    def like(self, a, device, body, canary, name=None):
        """A framed copy of the array or tensor a."""
        t = torch.as_tensor(np.ascontiguousarray(a)) if not isinstance(a, torch.Tensor) else a
        out = self.framed(t.shape, t.dtype, device, body, canary, name)
        out.copy_(t)
        return out

    def poison(self, t, body):
        """Refill the body of the framed tensor t (a workspace an object keeps across calls) with the byte body."""
        for _, raw, nbytes, _ in self.bufs:
            if raw.data_ptr() + FRAME == t.data_ptr():
                raw[FRAME:FRAME + nbytes].fill_(body)
                return
        raise KeyError("not a framed buffer")

    def frames_intact(self):
        """-> [(name, side, first changed byte offset from the body's start)] of every changed frame (printed); [] when all
        frames hold their byte."""
        bad = []
        for name, raw, nbytes, canary in self.bufs:
            r = raw.cpu().numpy()
            lo = np.flatnonzero(r[:FRAME] != canary)
            hi = np.flatnonzero(r[FRAME + nbytes:] != canary)
            if len(lo):
                bad.append((name, "left", int(lo[-1]) - FRAME))      # the changed byte nearest the body
            if len(hi):
                bad.append((name, "right", nbytes + int(hi[0])))
        for name, side, off in bad:
            print("frame changed: %s, %s frame, byte offset %d" % (name, side, off))
        return bad


class TorchShim(object):
    """`torch` for ops: forwards every attribute, serves empty / empty_like / zeros on the framer's devices framed."""

    def __init__(self, framer, poison):
        self._framer, self._poison = framer, poison

    def __getattr__(self, name):
        return getattr(torch, name)

    def _framed_device(self, device):
        if device is None:
            return None
        d = torch.device(device)
        return d if d.type in self._framer.devices else None

    def _make(self, size, dtype, device, body, what, **kw):
        shape = tuple(size[0]) if len(size) == 1 and isinstance(size[0], (tuple, list, torch.Size)) else tuple(size)
        dev = self._framed_device(device)
        if dev is None or kw.get("pin_memory") or kw.get("out") is not None:
            return getattr(torch, what)(*size, dtype=dtype, device=device, **kw)
        return self._framer.framed(shape, dtype or torch.get_default_dtype(), dev, body, CANARY, "%s%s" % (what, list(shape)))

    def empty(self, *size, dtype=None, device=None, **kw):
        return self._make(size, dtype, device, self._poison, "empty", **kw)

    def zeros(self, *size, dtype=None, device=None, **kw):
        return self._make(size, dtype, device, 0, "zeros", **kw)

    def empty_like(self, t, dtype=None, device=None, **kw):
        dev = t.device if device is None else device
        if self._framed_device(dev) is None or kw:
            return torch.empty_like(t, dtype=dtype, device=device, **kw)
        return self._make((t.shape,), dtype or t.dtype, dev, self._poison, "empty_like")


def to_host(x):
    """A result (tensor, array, number, None or a nested list / tuple / dict of them) -> the same with host arrays."""
    if isinstance(x, torch.Tensor):
        return x.detach().cpu().numpy().copy()
    if isinstance(x, (list, tuple)):
        return type(x)(to_host(v) for v in x)
    if isinstance(x, dict):
        return {k: to_host(v) for k, v in x.items()}
    return x


def bit_equal(a, b, where="out"):
    """Asserts a and b (to_host results) are bit-identical; NaN payloads count."""
    if isinstance(a, (list, tuple)):
        assert isinstance(b, (list, tuple)) and len(a) == len(b), where
        for k, (x, y) in enumerate(zip(a, b)):
            bit_equal(x, y, "%s[%d]" % (where, k))
    elif isinstance(a, dict):
        assert sorted(a) == sorted(b), where
        for k in a:
            bit_equal(a[k], b[k], "%s[%r]" % (where, k))
    elif isinstance(a, np.ndarray):
        assert a.shape == b.shape and a.dtype == b.dtype, where
        assert np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8)), where
    else:
        assert a == b or (a != a and b != b), where


def under_both_poisons(monkeypatch, mods, call, inputs=None, same=bit_equal):
    """Runs call(framer, poison, *inputs(framer, poison)) once with every poisoned byte 0xFF and once 0x00, `torch`
    replaced by a TorchShim in each module of mods; inputs builds the call's framed inputs (see framed_input).  Asserts
    every frame of both runs is intact and same(result 0xFF, result 0x00) (bit-identical by default); -> both results
    (to_host)."""
    res = []
    for poison in POISONS:
        framer = Framer()
        with monkeypatch.context() as mp:
            for m in (mods if isinstance(mods, (list, tuple)) else [mods]):
                mp.setattr(m, "torch", TorchShim(framer, poison))
            args = inputs(framer, poison) if inputs is not None else ()
            out = call(framer, poison, *args)
            torch.cuda.synchronize()
            res.append(to_host(out))
        assert framer.frames_intact() == [], "a frame changed under poison 0x%02X" % poison
    same(res[0], res[1])
    return res


def framed_input(framer, poison, a, device="cuda", name=None):
    """A framed device copy of the host array a, its frames holding the run's poison (NaN around float inputs in the 0xFF
    run, 0x00 and 0xFF around integer ones): a read past either end changes the result of one run."""
    return framer.like(a, device, poison, poison, name)
