"""Shared helpers of the C-boundary contract tests (tests/test_abi_contract_*.py): how the library hands results back.

include/flmr_maxsim.h promises that the caller owns every buffer, that compute calls are asynchronous on the stream they
are given, and that one corpus may serve concurrent searches through distinct workspaces.  The tests call the C entry
points directly, with explicit stream handles, and hold every call to the same call made plainly (default stream,
fresh buffers, inputs in place): bitwise.

* ``Guarded``: an output placed inside a larger allocation whose guard bands (each at least as large as the output
  and at least 64 KiB) and output are filled with a sentinel no kernel writes.  After a call the guards must be intact,
  every element of the documented output range must differ from the sentinel, and the elements outside it must not.
* ``Call``: one entry point with its inputs, the shapes of its outputs and the range of each output it must write;
  ``plain``, ``guarded``, ``gated`` and ``early_consumer`` run it the four ways the GPU module compares.
"""
from __future__ import annotations

import ctypes as C
import time
from dataclasses import dataclass, field
from typing import Callable, Dict, Optional

import numpy as np
import torch

GUARD_MIN_BYTES = 64 * 1024

# sentinel bit patterns, as the signed integers of the same width (every one is positive)
SENTINEL_BITS = {
    torch.float32: 0x7FBADBAD,             # a NaN with a payload no kernel produces
    torch.int64: 0x5A5A5A5A5A5A5A5A,
    torch.int32: 0x5A5A5A5A,
    torch.bfloat16: 0x7FAB,                # a bf16 NaN
    torch.float16: 0x7E5B,                 # an fp16 NaN
    torch.uint8: 0xA5,
}
_INT_VIEW = {torch.float32: torch.int32, torch.int64: torch.int64, torch.int32: torch.int32,
             torch.bfloat16: torch.int16, torch.float16: torch.int16, torch.uint8: torch.uint8}


def bits(t: torch.Tensor) -> torch.Tensor:
    """The tensor's storage as integers of its element width (NaN payloads and -0.0 compare bitwise)."""
    return t.view(_INT_VIEW[t.dtype])


def same_bits(a: torch.Tensor, b: torch.Tensor) -> bool:
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(bits(a), bits(b))


def guard_elems(n: int, dtype: torch.dtype) -> int:
    """Elements of each guard band of an n-element output: at least n and at least 64 KiB."""
    item = torch.empty((), dtype=dtype).element_size()
    return max(n, -(-GUARD_MIN_BYTES // item))


def ptr(t) -> C.c_void_p:
    """Device or host address of a tensor or numpy array (None stays NULL)."""
    if t is None:
        return C.c_void_p(None)
    if isinstance(t, np.ndarray):
        return t.ctypes.data_as(C.c_void_p)
    return C.c_void_p(t.data_ptr())


class Guarded:
    """An output of ``shape`` inside ``[guard | output | guard]``, all of it holding the sentinel."""

    def __init__(self, shape, dtype: torch.dtype, device="cuda"):
        self.shape, self.dtype = tuple(shape), dtype
        self.n = int(np.prod(self.shape)) if self.shape else 1
        self.g = guard_elems(self.n, dtype)
        self.buf = torch.empty(2 * self.g + self.n, dtype=dtype, device=device)
        self.fill()
        self.out = self.buf[self.g:self.g + self.n].view(self.shape)

    def fill(self) -> None:
        """Sentinel everywhere (on the current stream)."""
        bits(self.buf).fill_(SENTINEL_BITS[self.dtype])

    def fill_output(self) -> None:
        bits(self.buf[self.g:self.g + self.n]).fill_(SENTINEL_BITS[self.dtype])

    def check(self, written: Optional[torch.Tensor] = None, tag: str = "") -> None:
        """Both guards hold the sentinel bitwise; inside the output every element of ``written`` (bool, the output's
        shape; None: all of it) differs from the sentinel and every other element still holds it."""
        s = SENTINEL_BITS[self.dtype]
        b = bits(self.buf)
        lo, hi = b[:self.g], b[self.g + self.n:]
        bad_lo = (lo != s).nonzero()
        bad_hi = (hi != s).nonzero()
        assert bad_lo.numel() == 0, "%s: %d elements written before the output (last at -%d)" % (
            tag, bad_lo.numel(), self.g - int(bad_lo.max()))
        assert bad_hi.numel() == 0, "%s: %d elements written after the output (first at +%d)" % (
            tag, bad_hi.numel(), int(bad_hi.min()))
        o = bits(self.out)
        if written is None:
            written = torch.ones(self.shape, dtype=torch.bool, device=o.device)
        unwritten = written & (o == s)
        assert not unwritten.any(), "%s: %d of %d elements of the output range not written (first at %s)" % (
            tag, int(unwritten.sum()), int(written.sum()), tuple(unwritten.nonzero()[0].tolist()))
        stray = ~written & (o != s)
        assert not stray.any(), "%s: %d elements outside the output range written" % (tag, int(stray.sum()))


@dataclass
class Call:
    """One C entry point, ready to run.

    fn(ins, outs, stream) -> status: ``ins`` / ``outs`` map names to device tensors, ``stream`` is a cudaStream_t
    handle (an int, 0 = the legacy default stream).  Host inputs (``host``) are closed over by fn.
    outputs: name -> (shape, dtype); ``guarded(call, want, omit=name)`` passes an optional one as NULL.
    written: name -> bool mask of the elements the call must write (default: all of them).
    make_inputs(seed) -> another valid set of ``ins`` (the decoys and graph replays).
    close: name -> f(ins, got, want) -> bool for an output whose summation order is not fixed (fp32 atomics), held to
    a bound instead of bitwise.
    """
    name: str
    fn: Callable
    inputs: Dict[str, torch.Tensor]
    outputs: Dict[str, tuple]
    make_inputs: Callable
    host: Dict[str, np.ndarray] = field(default_factory=dict)
    written: Dict[str, torch.Tensor] = field(default_factory=dict)
    synchronous: bool = False          # flmr_plaid_decode: documented as synchronous on its stream
    close: Dict[str, Callable] = field(default_factory=dict)

    def run(self, ins, outs, stream) -> None:
        rc = self.fn(ins, outs, stream)
        assert rc == 0, "%s: status %d" % (self.name, rc)

    def empty_outputs(self):
        return {n: torch.empty(s, dtype=d, device="cuda") for n, (s, d) in self.outputs.items()}

    def plain(self, ins=None) -> Dict[str, torch.Tensor]:
        """The call made plainly: default stream, fresh buffers, inputs already in place."""
        torch.cuda.synchronize()
        outs = self.empty_outputs()
        self.run(self.inputs if ins is None else ins, outs, 0)
        torch.cuda.synchronize()
        return outs

    def compare(self, got: Dict[str, torch.Tensor], want: Dict[str, torch.Tensor], tag: str, ins=None) -> None:
        for n in want:
            if n not in got or got[n] is None:
                continue
            w = self.written.get(n)
            a, b = got[n], want[n]
            if n in self.close:
                assert self.close[n](self.inputs if ins is None else ins, a, b), (
                    "%s / %s: %s differs from the plain call beyond its bound" % (self.name, tag, n))
                continue
            if w is not None:
                a, b = a[w], b[w]
            assert same_bits(a, b), "%s / %s: %s differs from the plain call" % (self.name, tag, n)


def snapshot(ins: Dict[str, torch.Tensor], host: Dict[str, np.ndarray]):
    return ({n: t.clone() for n, t in ins.items()}, {n: a.copy() for n, a in host.items()})


def check_unchanged(call: Call, snap, tag: str) -> None:
    dev, host = snap
    for n, t in call.inputs.items():
        assert same_bits(t, dev[n]), "%s / %s: input %s was written" % (call.name, tag, n)
    for n, a in call.host.items():
        assert np.array_equal(a, host[n]), "%s / %s: host input %s was written" % (call.name, tag, n)


def guarded(call: Call, want: Dict[str, torch.Tensor], omit: Optional[str] = None) -> None:
    """Every output guarded, ``omit`` (an optional output) passed as NULL; default stream."""
    snap = snapshot(call.inputs, call.host)
    gs = {n: Guarded(s, d) for n, (s, d) in call.outputs.items()}
    outs = {n: (None if n == omit else g.out) for n, g in gs.items()}
    torch.cuda.synchronize()
    call.run(call.inputs, outs, 0)
    torch.cuda.synchronize()
    tag = "guarded" + ("" if omit is None else ", %s NULL" % omit)
    for n, g in gs.items():
        if n == omit:
            g.check(torch.zeros(g.shape, dtype=torch.bool, device="cuda"), "%s / %s / %s" % (call.name, tag, n))
        else:
            g.check(call.written.get(n), "%s / %s / %s" % (call.name, tag, n))
    call.compare({n: g.out for n, g in gs.items() if n != omit}, want, tag)
    check_unchanged(call, snap, tag)


def gate(stream: torch.cuda.Stream, cycles: int) -> torch.cuda.Event:
    """Hold ``stream`` with a spin kernel of ``cycles`` clock cycles; returns an event recorded behind it."""
    with torch.cuda.stream(stream):
        torch.cuda._sleep(int(cycles))
        ev = torch.cuda.Event()
        ev.record(stream)
    return ev


@dataclass
class GatedResult:
    call_seconds: float
    gate_done_at_return: bool


def gated(call: Call, S: torch.cuda.Stream, cycles: int, want: Dict[str, torch.Tensor], seed: int) -> GatedResult:
    """Late inputs on S: the inputs hold decoys; on S the gate, then the real inputs copied in, then the call, then
    clones of its outputs.  The clones must equal the plain call: any of the call's work not ordered after S's
    pending writes read the decoys.  Returns the host time of the call and whether the gate had ended on its return."""
    decoy = call.make_inputs(seed)
    ins = {n: decoy[n].clone() for n in call.inputs}
    gs = {n: Guarded(s, d) for n, (s, d) in call.outputs.items()}
    torch.cuda.synchronize()
    ev = gate(S, cycles)
    with torch.cuda.stream(S):
        for n, t in ins.items():
            t.copy_(call.inputs[n])
        t0 = time.perf_counter()
        call.run(ins, {n: g.out for n, g in gs.items()}, S.cuda_stream)
        dt = time.perf_counter() - t0
        done = ev.query()
        clones = {n: g.out.clone() for n, g in gs.items()}
    S.synchronize()
    torch.cuda.synchronize()
    for n, g in gs.items():
        g.check(call.written.get(n), "%s / late inputs / %s" % (call.name, n))
    call.compare(clones, want, "late inputs")
    return GatedResult(dt, done)


def early_consumer(call: Call, S: torch.cuda.Stream, cycles: int, want: Dict[str, torch.Tensor]) -> None:
    """The legacy default stream held by a gate; on S the outputs prefilled with the sentinel, the call, and clones of
    the outputs made at once.  The clones must be final: a launch that went to stream 0 has not run yet."""
    gs = {n: Guarded(s, d) for n, (s, d) in call.outputs.items()}
    torch.cuda.synchronize()
    gate(torch.cuda.default_stream(), cycles)
    with torch.cuda.stream(S):
        for g in gs.values():
            g.fill_output()
        call.run(call.inputs, {n: g.out for n, g in gs.items()}, S.cuda_stream)
        clones = {n: g.out.clone() for n, g in gs.items()}
    S.synchronize()
    torch.cuda.synchronize()
    call.compare(clones, want, "early consumer")


def graph_replay(call: Call, seeds=(101, 102)) -> None:
    """Capture the call after a warm-up, replay it twice with new input contents copied into the captured buffers;
    each replay must be bitwise the plain call on those contents."""
    ins = {n: t.clone() for n, t in call.inputs.items()}
    outs = call.empty_outputs()
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        call.run(ins, outs, s.cuda_stream)               # warm-up: sizes workspaces, loads modules
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        call.run(ins, outs, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    for seed in seeds:
        new = call.make_inputs(seed)
        for n, t in ins.items():
            t.copy_(new[n])
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        want = call.plain(new)
        call.compare(outs, want, "graph replay %d" % seed, ins=new)
    del g
