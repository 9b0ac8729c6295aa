"""What the GPU tests check every kernel result against: guarded output buffers, the rejected-call contract, error
metrics and the float64 error bounds shared by the stage tests.

Every output a kernel writes sits inside a buffer filled with a NaN sentinel, with guard regions on both sides: a store
outside the output changes a guard, an element the kernel skips keeps the sentinel.  The sentinels are non-canonical
NaNs that no kernel writes.  A rejected call must raise NativeError with its exact message, launch no kernel and write
nothing.
"""
import math

import pytest
import torch

from fadtk_b200 import _native

# dtype -> (integer view, sentinel bit pattern)
SENTINEL = {torch.float16: (torch.int16, 0x7E5A), torch.float32: (torch.int32, 0x7FC0FFEE)}


class Guarded:
    """A tensor of `shape` inside a sentinel-filled buffer: `guard` elements before it and `tail` (default: `guard`)
    after it.  `init` fills the tensor, which makes it an input whose contents intact_input() compares against."""

    def __init__(self, shape, dtype, device, guard, tail=None, init=None):
        self.n = math.prod(shape)
        self.guard = guard
        self.idt, self.bits = SENTINEL[dtype]
        self.buf = torch.empty(guard + self.n + (guard if tail is None else tail), dtype=dtype, device=device)
        self.buf.view(self.idt).fill_(self.bits)
        self.body = self.buf[guard:guard + self.n].view(shape)
        self.init = None
        if init is not None:
            self.body.copy_(init)
            self.init = self.body.clone()

    def _raw(self):
        if self.buf.is_cuda:
            torch.cuda.synchronize()
        return self.buf.view(self.idt)

    def guards_intact(self):
        raw = self._raw()
        return bool((raw[:self.guard] == self.bits).all()) and bool((raw[self.guard + self.n:] == self.bits).all())

    def fully_written(self):
        return not bool((self._raw()[self.guard:self.guard + self.n] == self.bits).any())

    def untouched(self):
        return bool((self._raw() == self.bits).all())

    def intact_input(self):
        return self.guards_intact() and torch.equal(self.body, self.init)

    def check(self, what="output"):
        """guards intact, every element written and finite -> the tensor"""
        assert self.guards_intact(), f"{what}: guard region overwritten"
        assert self.fully_written(), f"{what}: elements left unwritten"
        assert bool(torch.isfinite(self.body).all()), f"{what}: non-finite values"
        return self.body

    def ptr(self, kind):
        """the argument a call receives: the tensor ("ok"), None ("null"), or the buffer from one element past the
        tensor's start ("odd": misaligned for any vector access)"""
        return {"ok": self.body, "null": None, "odd": self.buf[self.guard + 1:]}[kind]


# ------------------------------------------------------------------------------------------------ rejected calls
def expect_rejected(engine, call, message, outs):
    """call(engine, outs) raises NativeError with exactly `message`, launches no kernel and leaves every Guarded in
    `outs` (the call may append the buffers it passes) untouched."""
    launches = engine.launches
    with pytest.raises(_native.NativeError) as exc:
        call(engine, outs)
    assert str(exc.value) == message, f"message {str(exc.value)!r}, want {message!r}"
    assert engine.launches == launches, "a rejected call launched a kernel"
    assert all(o.untouched() for o in outs), "a rejected call wrote output"


def on_fresh_engine(call):
    """The call made on a new engine of the same device, which has no model loaded; it must launch nothing there."""
    def run(engine, outs):
        fresh = _native.Engine(engine.device, 16)
        launches = fresh.launches
        try:
            call(fresh, outs)
        finally:
            after = fresh.launches
            fresh.close()
            assert after == launches, "a rejected call launched a kernel"
    return run


# ------------------------------------------------------------------------------------------------- error metrics
def rms_rel(got, ref):
    """rms |got - ref| / rms |ref|, ref float64"""
    return ((got.double() - ref).square().mean().sqrt() / ref.square().mean().sqrt()).item()


def report(tag, kind, what, line):
    print(f"\n[{tag} {kind}] {what}: {line}", flush=True)


def check_bound(kind, what, got, ref, bound, stats, ceilings):
    """|got - ref| <= bound element by element, and the rms relative error (the max |err| where ref is all zero) at
    most ceilings[kind] when there is one.  stats[kind] keeps [largest rms, largest max err / bound, the `what` of the
    largest rms].  -> (rms, max err / bound)"""
    err = (got.double() - ref).abs()
    r = err / bound
    ratio = r.max().item()
    worst = int(r.flatten().argmax())
    assert ratio <= 1.0, (f"{what}: max |err| / bound = {ratio:.3g} at flat index {worst} "
                          f"(got {got.flatten()[worst].item()!r}, want {ref.flatten()[worst].item()!r})")
    rms = rms_rel(got, ref) if bool(ref.abs().max() > 0) else err.max().item()
    if kind in ceilings:
        assert rms <= ceilings[kind], f"{what}: rms relative error {rms:.3g} above {ceilings[kind]:.3g}"
    st = stats.setdefault(kind, [0.0, 0.0, ""])
    if rms > st[0]:
        st[0], st[2] = rms, what
    st[1] = max(st[1], ratio)
    return rms, ratio


def report_stats(capsys, tag, stats, what):
    with capsys.disabled():
        for kind, (rms, ratio, w) in stats.items():
            report(tag, kind, what, f"largest rms rel err {rms:.3e} ({w}), max err / bound {ratio:.3f}")


def layer_metrics(got, x, ref):
    """(rms rel of the output, rms rel of the update out - x, max |err| / max |ref|) of a layer fed x"""
    rms = rms_rel(got, ref)
    upd = rms_rel(got.double() - x.double(), ref - x.double())
    mx = ((got.double() - ref).abs().max() / ref.abs().max()).item()
    return rms, upd, mx


def tap_metrics(got, ref):
    """(rms rel, centred rms rel, mean error / fluctuation rms) of [B, S, d] outputs against float64.  Centred: the
    per-(clip, channel) mean over positions removed from error and reference; the fluctuation is the centred
    reference, so the last two need S > 1."""
    err = got.double() - ref
    rms = (err.square().mean().sqrt() / ref.square().mean().sqrt()).item()
    ec = err - err.mean(1, keepdim=True)
    rc = ref - ref.mean(1, keepdim=True)
    fl = rc.square().mean().sqrt()
    centred = (ec.square().mean().sqrt() / fl).item()
    mean_err = (err.mean(1).square().mean().sqrt() / fl).item()
    return rms, centred, mean_err


# ---------------------------------------------------------------------------------------------- float64 bounds
def gemm_bound(S, sum_w, sum_a, K, b, y, r_a=0.0):
    """Error bound of the pre-activation output y = b + sum_j w_j a_j of a GEMM convolution with K reduction columns
    (b [Cout]; y, S, sum_a [B, Cout or 1, T]; sum_w [1, Cout, 1]), from the float64 sums the caller computes with the
    convolution's own taps, padding and stride: S = sum_j |w_j| |a_j|, sum_w = sum_j |w_j|, sum_a = sum_j |a_j|.
      * a_j rounded to fp16 by the kernel:                 r_a |a_j| (r_a = 2^-11; 0 when the operand is already the
                                                           fp16 value), + 2^-25 when it is fp16-subnormal
      * w_j the fp16 hi/lo pair of the fp32 weight:        2^-21 |w_j|, + 2^-25 for a subnormal lo part
      * fp32 accumulation of K products, and the bias add: K 2^-23 S + 2^-24 (|b| + |y|)
    so |got - y| <= (r_a + 2^-21 + K 2^-23) S + 2^-25 (sum_w + sum_a) + 2^-24 (|b| + |y|).  One wrong tap moves an
    output by |w_j a_j|, which random weights make comparable to S / sqrt(K) and so far above the bound.  The caller
    adds what the operand's own error contributes (sum_j |w_j| e_a_j) and its margin."""
    return (r_a + 2.0 ** -21 + K * 2.0 ** -23) * S + 2.0 ** -25 * (sum_w + sum_a) + 2.0 ** -24 * (b.abs()[None, :, None] + y.abs())


def ln_bound(y, e, g, beta, dim):
    """LayerNorm / GroupNorm (eps 1e-5) over `dim` of the float64 pre-norm values y, which carry errors e
    -> (normalised y, bound).  With mean m, rstd r: the mean moves by mean(e), the variance by
    dvar = 2 mean(|y - m| e) + mean(e)^2, r by half of that relatively (+ 2^-23 for its fp32 copy), and the fp32 affine
    adds 2^-22 (|out| + |beta|):
      |d out| <= |g| r (e + mean(e) + 2^-24 |m|) + |g| |y - m| r (dvar / (2 (var + eps)) + 2^-23) + 2^-22 (|out| + |beta|)"""
    m = y.mean(dim, keepdim=True)
    yc = y - m
    var = yc.square().mean(dim, keepdim=True)
    r = 1.0 / torch.sqrt(var + 1e-5)
    me = e.mean(dim, keepdim=True)
    dvar = 2 * (yc.abs() * e).mean(dim, keepdim=True) + me.square()
    yn = yc * r * g + beta
    return yn, (g.abs() * r * (e + me + 2.0 ** -24 * m.abs()) + g.abs() * yc.abs() * r * (dvar / (2 * (var + 1e-5)) + 2.0 ** -23)
                + 2.0 ** -22 * (yn.abs() + beta.abs()))


def gelu_out(y, e, fp16):
    """GELU of the float64 y, which carries errors e -> (GELU(y), bound): 1.13 (GELU's largest slope) e + 2^-22 |out|
    for its fp32 evaluation; an fp16 output adds 2^-11 (|out| + e) + 2^-25."""
    out = torch.nn.functional.gelu(y)
    e = 1.13 * e + 2.0 ** -22 * out.abs()
    if fp16:
        e = e + 2.0 ** -11 * (out.abs() + e) + 2.0 ** -25
    return out, e
