"""TV-L1 optical flow on the GPU (csrc/flow.cu): the grey conversion, the batched solver and the 8-bit flow frames
that the reference's TV-L1 flow databases store.

    g = grey(frames)                       # uint8 [N, H, W, 3] RGB on the GPU -> float32 [N, H, W] (Pillow's 'L')
    flow, iters = tvl1(g[:-1], g[1:])      # float32 [P, 2, H, W] (u1 horizontal, u2 vertical), int32 [P, S, 5]
    frames = quantise(flow)                # uint8 [P, H, W, 3]: R = q(u1), G = q(u2), B = 128

The solver's parameters are fixed (include/coclr_b200.h): zoom factor 0.5, at most 5 scales, 5 warps, lambda 0.15,
theta 0.3, tau 0.25, epsilon 0.01, at most 300 iterations per warp.  Convergence is decided per pair on the device,
so a pair's flow is bit-identical whatever batch it is solved in.  The workspace is allocated per call.
"""
import ctypes as C

import torch

from . import lib as L

BOUND = 20.0          # flow frames truncate at +-BOUND px: q(f) = clamp(floor((f + 20) * 255 / 40 + 0.5), 0, 255)
ZERO_BYTE = 128       # the third channel, q(0)
# The byte layout of a stored flow frame (the reference does not fix it): channel -> what it holds
LAYOUT = ("u1 (horizontal)", "u2 (vertical)", "zero")
WARPS = 5
MAX_BATCH = 65535     # pairs (frames for grey) per library call (COCLR_FLOW_MAX_BATCH); larger batches run in chunks


def _planes(t, name, dims):
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float32 or t.dim() != dims:
        raise ValueError("%s must be a CUDA float32 tensor with %d dimensions" % (name, dims))
    return t.contiguous()


def scales(h, w):
    """Pyramid levels of an h x w solve."""
    n = L.load().coclr_tvl1_scales(h, w)
    if n < 0:
        raise ValueError("invalid frame size %d x %d" % (h, w))
    return n


def grey(frames):
    """uint8 [N, H, W, 3] RGB frames on the GPU (rows and frames may be strided, pixels packed) -> float32 [N, H, W],
    Pillow's convert('L') bit for bit, as floats 0..255."""
    if (not isinstance(frames, torch.Tensor) or not frames.is_cuda or frames.dtype != torch.uint8 or frames.dim() != 4
            or frames.shape[3] != 3 or frames.stride(3) != 1 or frames.stride(2) != 3):
        raise ValueError("frames must be a CUDA uint8 [N, H, W, 3] tensor with packed pixels")
    n, h, w, _ = frames.shape
    out = torch.empty(n, h, w, dtype=torch.float32, device=frames.device)
    for a in range(0, n, MAX_BATCH):
        m = min(MAX_BATCH, n - a)
        L.check(L.load().coclr_flow_grey(L.dptr(frames[a:]), m, h, w, frames.stride(0), frames.stride(1),
                                         L.dptr(out[a:]), L.stream_ptr()), "coclr_flow_grey")
    return out


def tvl1(i0, i1):
    """TV-L1 flow of P pairs: i0, i1 float32 [P, H, W] on the GPU.  Returns (flow float32 [P, 2, H, W] with
    I1(x + flow) ~ I0(x), iterations int32 [P, scales, WARPS]).  More than MAX_BATCH pairs are solved in consecutive
    chunks, which gives the same result: each pair's solve is independent of the others in its batch."""
    i0, i1 = _planes(i0, "i0", 3), _planes(i1, "i1", 3)
    if i0.shape != i1.shape or i0.device != i1.device:
        raise ValueError("i0 and i1 must have the same shape and device, got %s and %s" % (tuple(i0.shape),
                                                                                        tuple(i1.shape)))
    P, H, W = i0.shape
    flow = torch.empty(P, 2, H, W, dtype=torch.float32, device=i0.device)
    iters = torch.zeros(P, scales(H, W), WARPS, dtype=torch.int32, device=i0.device)
    if P == 0:
        return flow, iters
    lib = L.load()
    chunk = min(P, MAX_BATCH)
    work = torch.empty(lib.coclr_tvl1_work_bytes(chunk, H, W), dtype=torch.uint8, device=i0.device)
    for a in range(0, P, chunk):
        m = min(chunk, P - a)
        t = L.Tvl1(m, H, W, L.dptr(i0[a:]), L.dptr(i1[a:]), L.dptr(flow[a:]), L.dptr(iters[a:]), L.dptr(work),
                   work.numel())
        L.check(lib.coclr_tvl1(C.byref(t), L.stream_ptr()), "coclr_tvl1")
    return flow, iters


def quantise(flow):
    """float32 [P, 2, H, W] flow -> uint8 [P, H, W, 3] frames (LAYOUT)."""
    flow = _planes(flow, "flow", 4)
    if flow.shape[1] != 2:
        raise ValueError("flow must be [P, 2, H, W]")
    P, _, H, W = flow.shape
    out = torch.empty(P, H, W, 3, dtype=torch.uint8, device=flow.device)
    for a in range(0, P, MAX_BATCH):
        L.check(L.load().coclr_flow_quantise(L.dptr(flow[a:]), min(MAX_BATCH, P - a), H, W, L.dptr(out[a:]),
                                             L.stream_ptr()), "coclr_flow_quantise")
    return out


# --- the solver's stages, one at a time (for tests) -------------------------------------------------------------------

def zoom_out(x, hc, wc):
    """One pyramid level down: Gaussian, then bicubic sampling, float32 [P, H, W] -> [P, hc, wc]."""
    x = _planes(x, "x", 3)
    P, H, W = x.shape
    tmp = torch.empty(2, P, H, W, dtype=torch.float32, device=x.device)
    out = torch.empty(P, hc, wc, dtype=torch.float32, device=x.device)
    L.check(L.load().coclr_flow_zoom_out(L.dptr(x), P, H, W, L.dptr(tmp), L.dptr(out), hc, wc, L.stream_ptr()),
            "coclr_flow_zoom_out")
    return out


def zoom_in(flow, h, w):
    """Coarse flow float32 [P, 2, Hc, Wc] -> [P, 2, h, w], u1 scaled by w / Wc and u2 by h / Hc."""
    flow = _planes(flow, "flow", 4)
    P, _, hc, wc = flow.shape
    out = torch.empty(P, 2, h, w, dtype=torch.float32, device=flow.device)
    L.check(L.load().coclr_flow_zoom_in(L.dptr(flow), P, hc, wc, L.dptr(out), h, w, L.stream_ptr()),
            "coclr_flow_zoom_in")
    return out


def warp(i0, i1, flow):
    """float32 [6, P, H, W]: I1x, I1y (centred gradients of i1), I1x and I1y warped at x + flow, g, rho_c."""
    i0, i1, flow = _planes(i0, "i0", 3), _planes(i1, "i1", 3), _planes(flow, "flow", 4)
    P, H, W = i0.shape
    out = torch.empty(6, P, H, W, dtype=torch.float32, device=i0.device)
    L.check(L.load().coclr_flow_warp(L.dptr(i0), L.dptr(i1), L.dptr(flow), P, H, W, L.dptr(out), L.stream_ptr()),
            "coclr_flow_warp")
    return out


def iterate(warped, flow, dual, n):
    """n primal-dual iterations on warp()'s planes, updating flow [P, 2, H, W] and dual [P, 4, H, W] in place;
    returns the iterations each pair ran (int32 [P]) before it converged or n ran out."""
    warped = _planes(warped, "warped", 4)
    for t, name in ((flow, "flow"), (dual, "dual")):
        if _planes(t, name, 4) is not t:
            raise ValueError("%s must be contiguous (it is updated in place)" % name)
    _, P, H, W = warped.shape
    lib = L.load()
    work = torch.empty(lib.coclr_flow_iterate_work_bytes(P, H, W), dtype=torch.uint8, device=flow.device)
    iters = torch.empty(P, dtype=torch.int32, device=flow.device)
    L.check(lib.coclr_flow_iterate(L.dptr(warped), L.dptr(flow), L.dptr(dual), P, H, W, n, L.dptr(iters),
                                   L.dptr(work), L.stream_ptr()), "coclr_flow_iterate")
    return iters
