"""Thin Python wrappers (torch tensors -> raw pointers) over the C ABI. No autograd here; the
encoder-level autograd.Function lives in moco.py / engine.py."""
import ctypes as C

import torch

from . import lib as L


class Geometry:
    """Conv / pool geometry (kernel, stride, padding) per (t, h, w)."""

    def __init__(self, k, s=(1, 1, 1), p=(0, 0, 0)):
        self.k, self.s, self.p = tuple(k), tuple(s), tuple(p)

    @property
    def taps(self):
        return self.k[0] * self.k[1] * self.k[2]

    def out_dims(self, T, H, W):
        return tuple((d + 2 * p - k) // s + 1 for d, k, s, p in zip((T, H, W), self.k, self.s, self.p))

    def c(self, transposed=0):
        return L.Geom(self.k[0], self.k[1], self.k[2], self.s[0], self.s[1], self.s[2],
                      self.p[0], self.p[1], self.p[2], int(transposed))


class Planes:
    """A split-precision channels-last activation: two 16-bit planes [B,T,H,W,C] with hi + lo ~= value."""

    def __init__(self, shape, bf16, device, lo=True, zero=False):
        dt = torch.bfloat16 if bf16 else torch.float16
        self.bf16 = int(bool(bf16))
        mk = torch.zeros if zero else torch.empty
        self.hi = mk(shape, dtype=dt, device=device)
        self.lo = mk(shape, dtype=dt, device=device) if lo else None

    @property
    def ld(self):
        return self.hi.shape[-1]

    def value(self):
        v = self.hi.float()
        return v + self.lo.float() if self.lo is not None else v

    def src(self, coff, Cc, T, H, W):
        return L.Src(L.dptr(self.hi), L.dptr(self.lo), self.ld, coff, Cc, T, H, W)


def split_into(x, planes, coff=0, Cc=None, scale=None, shift=None, relu=False, out_coff=0, twin=None):
    """planes[..., out_coff:out_coff+C] = split(relu?(scale*x[..., coff:coff+C]+shift)); x fp32 rows.
    twin: optional bf16 Planes of the same shape receiving the same values."""
    Cc = Cc or x.shape[-1]
    M = x.numel() // x.shape[-1]
    p = L.Split(L.dptr(x), x.shape[-1], coff, Cc, M, L.dptr(scale), L.dptr(shift), int(bool(relu)),
                L.dptr(planes.hi), L.dptr(planes.lo), planes.ld, out_coff, planes.bf16,
                L.dptr(twin.hi) if twin is not None else None, L.dptr(twin.lo) if twin is not None else None,
                L.BnFinalize())
    L.check(L.load().coclr_affine_split(C.byref(p), L.num_sms(), L.stream_ptr()), "coclr_affine_split")
    return planes


def packed_layout(N, Kreal):
    lib = L.load()
    bn, nt = C.c_int(0), C.c_int(0)
    nbytes = lib.coclr_conv_packed_bytes(N, Kreal, C.byref(bn), C.byref(nt))
    return int(nbytes), bn.value, nt.value


class PackedWeights:
    """fp16/bf16 hi/lo swizzled tile images of one conv weight for one GEMM orientation."""

    def __init__(self, Cout, Cin, taps, cpad, mode, bf16, device):
        self.Cout, self.Cin, self.taps, self.cpad, self.mode, self.bf16 = Cout, Cin, taps, cpad, mode, int(bf16)
        self.N = Cout if mode == 0 else Cin
        self.Kreal = taps * cpad
        nbytes, self.BN, self.n_tiles = packed_layout(self.N, self.Kreal)
        self.wpk = torch.empty(nbytes, dtype=torch.uint8, device=device)
        self.unscale = torch.empty(self.BN * self.n_tiles, dtype=torch.float32, device=device)

    def pack(self, w):
        """w: PyTorch conv weight [Cout, Cin, kt, kh, kw] fp32 (contiguous, CUDA)."""
        assert w.is_contiguous() and w.dtype == torch.float32
        p = L.Pack(L.dptr(w), self.Cout, self.Cin, self.taps, self.cpad, self.mode, self.bf16,
                   L.dptr(self.wpk), L.dptr(self.unscale))
        L.check(L.load().coclr_pack_weights(C.byref(p), L.stream_ptr()), "coclr_pack_weights")
        return self


def make_conv(src, a_bf16, geom_c, B, dst_dims, pw, dst, dst_coff=0, accumulate=False, stats_sum=None,
              stats_sq=None, npass=3, out_scale=None):
    Td, Hd, Wd = dst_dims
    return L.Conv(src, geom_c, B, Td, Hd, Wd, pw.Kreal, L.dptr(pw.wpk), L.dptr(pw.unscale),
                  pw.N, pw.BN, pw.n_tiles, L.dptr(dst), dst.shape[-1], dst_coff, int(bool(accumulate)),
                  L.dptr(stats_sum), L.dptr(stats_sq), npass, int(a_bf16), pw.bf16, L.dptr(out_scale))


def conv_igemm(src, a_bf16, geom_c, B, dst_dims, pw, dst, dst_coff=0, accumulate=False, stats=None, npass=3,
               out_scale=None):
    """Run the implicit-GEMM conv. src: L.Src of 16-bit planes; dst: [B,Td,Hd,Wd,ld] fp32."""
    ssum = stats[:pw.N] if stats is not None else None
    ssq = stats[pw.N:] if stats is not None else None
    p = make_conv(src, a_bf16, geom_c, B, dst_dims, pw, dst, dst_coff, accumulate, ssum, ssq, npass, out_scale)
    L.check(L.load().coclr_conv_igemm(C.byref(p), L.num_sms(), L.stream_ptr()), "coclr_conv_igemm")


def conv_wgrad(src, src_bf16, geom_c, dy_src, dy_bf16, B, dst_dims, Cout, Cin_real, dw, npass=3, splits=1,
               out_scale=None, workspace=True):
    """workspace: fp32 tensor of at least coclr_wgrad_ws_floats floats, which the TMA-staged kernel needs (partial sums
    by plain stores + one reduction launch); True allocates one of the size the shape asks for, None runs the call on
    the gather kernel."""
    Td, Hd, Wd = dst_dims
    p = L.Wgrad(src, geom_c, dy_src, B, Td, Hd, Wd, Cout, Cin_real, L.dptr(dw), npass, int(dy_bf16), int(src_bf16),
                splits, L.dptr(out_scale))
    if workspace is True:
        need = int(L.load().coclr_wgrad_ws_floats(C.byref(p)))
        workspace = torch.empty(max(need, 4), dtype=torch.float32, device=dw.device)
    if workspace is not None:
        p.ws, p.ws_floats = L.dptr(workspace).value, workspace.numel()
    L.check(L.load().coclr_conv_wgrad(C.byref(p), L.stream_ptr()), "coclr_conv_wgrad", (C.byref(p),))
    return workspace
