"""NaN guard bands around kernel operands and per-element error bounds, shared by the float64-reference kernel tests.

Operands and outputs live inside larger buffers filled with NaN: NaN rows before and after, and NaN columns past the
leading dimension where the API allows a stride (contiguous operands are slices of a flat NaN buffer).  A read outside
an operand carries a NaN into some output; after a launch every element of the output view must be finite and every
element outside it bitwise unchanged, which catches both unwritten elements and stray writes."""
import math

import torch

NAN = float("nan")


class Guarded:
    """`view` ([rows, cols]) sits at row `pre` of a NaN-filled [pre + rows + post, ld] buffer, ld = cols rounded up
    to 8 plus `pad` columns, or the given `ld` with the view at column `col`.  `flat=True`: a contiguous tensor of any
    shape inside a flat NaN buffer instead."""

    def __init__(self, shape, dtype, dev, *, pre=3, post=5, pad=8, flat=False, ld=None, col=0):
        assert pad % 8 == 0
        self.dtype = dtype
        if flat:
            n = math.prod(shape)
            self.buf = torch.full((8 * pre + n + 8 * post,), NAN, dtype=dtype, device=dev)
            self.view = self.buf[8 * pre:8 * pre + n].view(shape)
        else:
            rows, cols = shape
            if ld is None:
                ld = -(-cols // 8) * 8 + pad
            assert col + cols <= ld
            self.buf = torch.full((pre + rows + post, ld), NAN, dtype=dtype, device=dev)
            self.view = self.buf[pre:pre + rows, col:col + cols]
        assert self.view.data_ptr() % 16 == 0 or col, "views at column 0 start 16-byte aligned"

    def fill(self, values):
        self.view.copy_(values)
        return self

    def snapshot(self):
        self._snap = self.buf.clone()
        return self

    def check(self, name):
        """Inside the view: finite.  Outside: bitwise what it was at snapshot()."""
        # in slabs of the first dim: isfinite's temporaries of a multi-GB view would be several times its size
        step = max(1, (1 << 26) * max(1, self.view.shape[0]) // max(1, self.view.numel()))
        assert all(torch.isfinite(self.view[i:i + step]).all() for i in range(0, self.view.shape[0], step)), \
            f"{name}: unwritten or non-finite output elements"
        ity = {2: torch.int16, 4: torch.int32, 8: torch.int64}[self.buf.element_size()]
        buf, snap = self.buf.view(ity), self._snap.view(ity)
        off = self.view.storage_offset() - self.buf.storage_offset()
        if self.buf.dim() == 2 and self.view.dim() == 2 and self.view.stride() == self.buf.stride():
            # a window of rows r0:r1 and columns c0:c1: compare the four regions around it (no index tensors, so
            # multi-GB outputs stay affordable)
            ld = self.buf.shape[1]
            r0, c0 = divmod(off, ld)
            r1, c1 = r0 + self.view.shape[0], c0 + self.view.shape[1]
            regions = [(slice(None, r0), slice(None)), (slice(r1, None), slice(None)),
                       (slice(r0, r1), slice(None, c0)), (slice(r0, r1), slice(c1, None))]
            n_bad = sum((buf[r] != snap[r]).sum().item() for r in regions)
        else:
            idx = torch.arange(self.buf.numel(), device=self.buf.device).view(self.buf.shape)
            inside = idx.as_strided(self.view.shape, self.view.stride(), off)
            outside = torch.ones(self.buf.numel(), dtype=torch.bool, device=self.buf.device)
            outside[inside.reshape(-1)] = False
            n_bad = (buf.reshape(-1)[outside] != snap.reshape(-1)[outside]).sum().item()
        assert n_bad == 0, f"{name}: {n_bad} elements outside the output view were written"


def _check_bound(out, ref, bound, name, family, l2=2 ** -8):
    """Every element within `bound`, relative L2 within `l2`; prints the margin (run with -s to see it)."""
    out = out.double()
    err = (out - ref).abs()
    ratio = (err / bound).max().item()
    rel_l2 = (err.norm() / ref.norm().clamp_min(1e-300)).item()
    print(f"[{family}] {name}: max err/bound {ratio:.3f}, rel L2 {rel_l2:.3e}")
    assert torch.isfinite(out).all(), f"{name}: non-finite output"
    n_bad = (err > bound).sum().item()
    assert n_bad == 0, f"{name}: {n_bad}/{err.numel()} elements beyond the derived bound (worst ratio {ratio:.3f})"
    assert rel_l2 <= l2, f"{name}: relative L2 error {rel_l2:.3e} > {l2:.3e}"
