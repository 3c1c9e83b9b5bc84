"""Output fences, comparisons and the kernel-name profiler shared by the GPU edge files (test_gpu_gemm_edges.py,
test_gpu_pooling_edges.py)."""
import numpy as np
import torch

SENT16 = 0x7FA5          # a NaN payload no kernel writes
SENT32 = 0x7FA5A5A5


def equal(got, want, what):
    got = np.asarray(got)
    if np.array_equal(got, want):
        return
    bad = ~(got == want)
    i = tuple(np.argwhere(bad)[0])
    raise AssertionError("{}: {} of {} elements differ; first at {}: got {!r}, want {!r}".format(
        what, int(bad.sum()), bad.size, i, got[i], want[i]))


def within(got, want, bound, what):
    """|got - want| <= bound elementwise (NaN where want is NaN must be NaN); returns the largest error / bound.  On failure
    names the worst element."""
    got = np.asarray(got, dtype=np.float64)
    both = np.isnan(got) & np.isnan(want)
    err = np.where(both, 0.0, np.abs(got - want))
    bad = ~(err <= bound)
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(err == 0, 0.0, err / bound)
    ratio = np.where(np.isnan(ratio), np.inf, ratio)
    if bad.any():
        i = np.unravel_index(int(np.argmax(np.where(bad, ratio, -1.0))), ratio.shape)
        raise AssertionError("{}: {} elements outside the bound; worst at {}: got {!r}, want {!r}, bound {!r}".format(
            what, int(bad.sum()), tuple(int(j) for j in i), got[i], want[i], bound[i]))
    return float(ratio.max()) if ratio.size else 0.0


class Fenced:
    """A view inside a larger buffer that starts out as a sentinel bit pattern."""

    def __init__(self, shape, dtype, index):
        self.buf = torch.empty(shape, dtype=dtype, device="cuda")
        self.sent = SENT16 if dtype == torch.bfloat16 else SENT32
        self.bits = self.buf.view(torch.int16 if dtype == torch.bfloat16 else torch.int32)
        self.bits.fill_(self.sent)
        self.view = self.buf[index]
        self.outside = torch.ones(shape, dtype=torch.bool, device="cuda")
        self.outside[index] = False

    def check(self, what):
        n = int((self.bits[self.outside] != self.sent).sum())
        assert n == 0, "{}: {} elements outside the output were written".format(what, n)

    def numpy(self):
        return self.view.float().cpu().numpy()


def profiled(run, pattern):
    """Calls run() under torch.profiler and returns the 'name<args>' strings of the kernels it launched whose names match
    the compiled regex `pattern` (groups: name, template arguments).  A short profiler session now and then returns no
    kernel records at all (seen on the H100: 2 of about 120 sessions); every caller launches a matching kernel, so an
    empty capture is the profiler's miss and is taken again, up to three times.  run() only rewrites the same outputs
    and checks them again."""
    seen = set()
    for _ in range(3):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            run()
            torch.cuda.synchronize()
        for e in prof.events():
            m = pattern.search(e.name)
            if m:
                seen.add("{}<{}>".format(m.group(1), m.group(2).replace(" ", "")))
        if seen:
            break
    return seen
