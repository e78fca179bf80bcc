"""Specification (CPU, torch) of the strided data-gradient as per-parity-class stride-1 gathers -- the form in which the
tensor-core kernel can feed it through im2col-mode TMA tensor maps.  TEST INFRASTRUCTURE / design note, not product code.

Why: ``din[y, x] = sum_{r, s} dout[(y + pad - r) / st, (x + pad - s) / st] w[r, s]`` only has the taps with
``(y + pad - r) % st == 0``; a tensor map cannot express "every st-th tap", so ``igemm_tc.cu`` still stages strided dgrad with
cp.async.  Splitting the output pixels into the st x st
classes ``(ey, ex) = ((y + pad) % st, (x + pad) % st)`` turns every class into a *stride-1* correlation of ``dout`` with the
sub-kernel ``w[ey::st, ex::st]``:

    y = st * iy + y0,  y0 = (ey - pad) mod st,  cy = (y0 + pad - ey) / st,   taps r = ey + st * tr, tr = 0 .. Tr - 1
    din[y, x] = sum_{tr, ts} dout[iy + cy - tr, ix + cx - ts] * w[ey + st tr, ex + st ts]          (zero outside dout)

which is an im2col load over ``dout`` with lower corner ``L = c - (T - 1)`` per axis, filter offset ``(T - 1) - t``, traversal
stride 1 and an upper corner that makes the bounding box hold exactly the class's pixel count:  ``U = Hc - Ho + L``.
``class_plan`` returns those numbers; ``dgrad_by_classes`` evaluates the data gradient through a faithful emulation of the
im2col traversal (``im2col_rows``, the semantics of CUDA's im2col-mode tensor maps) and
``tests/test_strided_dgrad_spec.py`` checks it against ``torch.nn.grad.conv2d_input``.
"""
import torch


def class_plan(H, Ho, R, stride, pad, e):
    """Per axis: (first pixel y0, number of class pixels Hc, taps Tr, lower corner L, upper corner U, c) or None if empty."""
    y0 = (e - pad) % stride
    if y0 >= H or e >= R:
        return None if y0 >= H else dict(y0=y0, Hc=-(-(H - y0) // stride), T=0, L=0, U=0, c=0)
    Hc = -(-(H - y0) // stride)
    T = -(-(R - e) // stride)
    c = (y0 + pad - e) // stride
    L = c - (T - 1)
    return dict(y0=y0, Hc=Hc, T=T, L=L, U=Hc - Ho + L, c=c)


def im2col_rows(t, lower, upper, start, offsets, pixels):
    """Emulation of ``cp.async.bulk.tensor.4d...im2col`` on an NHWC tensor ``t`` [N, H, W, C] with traversal stride 1: starting at
    base pixel ``start = (n, h, w)`` (coordinates inside the bounding box [lower, dim - 1 + upper]) walk ``pixels`` base pixels
    along W, then H, then N; each row is the tensor element at base + ``offsets`` (zero outside the tensor / past the end)."""
    N, H, W, C = t.shape
    (lh, lw), (uh, uw) = lower, upper
    bh, bw = H + uh - lh, W + uw - lw               # base pixels per image along h / w
    n, h, w = start
    lin = (n * bh + (h - lh)) * bw + (w - lw)
    out = torch.zeros(pixels, C, dtype=t.dtype)
    for i in range(pixels):
        k = lin + i
        nn, rem = divmod(k, bh * bw)
        hh, ww = divmod(rem, bw)
        y, x = hh + lh + offsets[0], ww + lw + offsets[1]
        if nn < N and 0 <= y < H and 0 <= x < W:
            out[i] = t[nn, y, x]
    return out


def dgrad_by_classes(dout, w, in_hw, stride, pad, tile=128):
    """``conv2d_input`` for NCHW ``dout`` [N, Co, Ho, Wo] and OIHW ``w`` via per-class im2col GEMMs (tile rows at a time)."""
    N, Co, Ho, Wo = dout.shape
    _, Ci, R, S = w.shape
    H, W = in_hw
    d_nhwc = dout.permute(0, 2, 3, 1).contiguous()
    din = torch.zeros(N, Ci, H, W, dtype=dout.dtype)
    for ey in range(stride):
        py = class_plan(H, Ho, R, stride, pad, ey)
        if py is None:
            continue
        for ex in range(stride):
            px = class_plan(W, Wo, S, stride, pad, ex)
            if px is None or py["T"] == 0 or px["T"] == 0:
                continue   # no tap reaches this class: its gradient is zero
            M = N * py["Hc"] * px["Hc"]
            lower, upper = (py["L"], px["L"]), (py["U"], px["U"])
            for m0 in range(0, M, tile):
                rows = min(tile, M - m0)
                n0, rem = divmod(m0, py["Hc"] * px["Hc"])
                iy0, ix0 = divmod(rem, px["Hc"])
                acc = torch.zeros(rows, Ci, dtype=dout.dtype)
                for tr in range(py["T"]):
                    for ts in range(px["T"]):
                        A = im2col_rows(d_nhwc, lower, upper, (n0, iy0 + py["L"], ix0 + px["L"]),
                                        (py["T"] - 1 - tr, px["T"] - 1 - ts), rows)          # [rows, Co]
                        acc += A @ w[:, :, ey + stride * tr, ex + stride * ts]                   # [Co, Ci]
                for i in range(rows):   # epilogue scatter: class pixel (n, iy, ix) -> (n, y0 + st iy, x0 + st ix)
                    n, rem = divmod(m0 + i, py["Hc"] * px["Hc"])
                    iy, ix = divmod(rem, px["Hc"])
                    din[n, :, py["y0"] + stride * iy, px["y0"] + stride * ix] = acc[i]
    return din
