"""float64 numpy oracle of the TV-L1 flow of coclr_b200.flow (include/coclr_b200.h gives the method), vectorised over
pixels, one pair at a time, plus the host references of the grey conversion and the quantisation.

    flow, iters = tvl1(i0, i1)          # i0, i1 [H, W]; flow [2, H, W] float64, iters [scales, 5]
"""
import math

import numpy as np

ETA, MAX_SCALES, MIN_SIDE, WARPS, MAX_ITERS = 0.5, 5, 16, 5, 300
LAMBDA, THETA, TAU, EPSILON, GRAD_ZERO = 0.15, 0.3, 0.25, 0.01, 1e-10
BOUND = 20.0


def grey(rgb):
    """uint8 [..., 3] -> uint8 [...]: Pillow's convert('L')."""
    r, g, b = (rgb[..., c].astype(np.int64) for c in range(3))
    return ((19595 * r + 38470 * g + 7471 * b + 0x8000) >> 16).astype(np.uint8)


def quantise(flow):
    """float32 [P, 2, H, W] -> uint8 [P, H, W, 3] in float32 arithmetic."""
    f = np.asarray(flow, np.float32)
    q = np.floor((f + np.float32(BOUND)) * np.float32(255.0 / (2 * BOUND)) + np.float32(0.5))
    q = np.clip(q, 0, 255).astype(np.uint8)
    out = np.full(f.shape[:1] + f.shape[2:] + (3,), 128, np.uint8)
    out[..., 0], out[..., 1] = q[:, 0], q[:, 1]
    return out


def sizes(h, w):
    out = [(h, w)]
    while len(out) < MAX_SCALES:
        hc, wc = int(out[-1][0] * ETA + 0.5), int(out[-1][1] * ETA + 0.5)
        if min(hc, wc) < MIN_SIDE:
            break
        out.append((hc, wc))
    return out


def gaussian_taps():
    sigma = 0.6 * math.sqrt(1.0 / (ETA * ETA) - 1.0)
    r = int(math.ceil(3 * sigma))
    k = np.arange(-r, r + 1, dtype=np.float64)
    w = np.exp(-0.5 * k * k / (sigma * sigma))
    return w / w.sum(), r


def blur(img):
    w, r = gaussian_taps()
    h, wd = img.shape
    xs, ys = np.arange(wd), np.arange(h)
    tmp = sum(w[k + r] * img[:, np.clip(xs + k, 0, wd - 1)] for k in range(-r, r + 1))
    return sum(w[k + r] * tmp[np.clip(ys + k, 0, h - 1), :] for k in range(-r, r + 1))


def keys(t):
    """Keys a = -0.5 weights [4, ...] of neighbours -1, 0, 1, 2 at fractional offset t."""
    t2, t3 = t * t, t * t * t
    return np.stack([-0.5 * t3 + t2 - 0.5 * t, 1.5 * t3 - 2.5 * t2 + 1.0, -1.5 * t3 + 2.0 * t2 + 0.5 * t,
                     0.5 * t3 - 0.5 * t2])


def bicubic(img, sx, sy):
    """img [H, W] sampled at float positions sx, sy (same shape), neighbour indices clamped."""
    h, w = img.shape
    fx, fy = np.floor(sx), np.floor(sy)
    wx, wy = keys(sx - fx), keys(sy - fy)
    x0, y0 = fx.astype(np.int64), fy.astype(np.int64)
    out = np.zeros(sx.shape)
    for j in range(4):
        yy = np.clip(y0 - 1 + j, 0, h - 1)
        row = sum(wx[i] * img[yy, np.clip(x0 - 1 + i, 0, w - 1)] for i in range(4))
        out += wy[j] * row
    return out


def zoom_out(img, hc, wc):
    h, w = img.shape
    y, x = np.mgrid[0:hc, 0:wc].astype(np.float64)
    return bicubic(blur(img), x * (w / wc), y * (h / hc))


def zoom_in(flow, h, w):
    _, hc, wc = flow.shape
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    sx, sy = x * (wc / w), y * (hc / h)
    return np.stack([bicubic(flow[0], sx, sy) * (w / wc), bicubic(flow[1], sx, sy) * (h / hc)])


def gradient(img):
    """Centred differences with clamp-to-edge."""
    h, w = img.shape
    xs, ys = np.arange(w), np.arange(h)
    gx = 0.5 * (img[:, np.minimum(xs + 1, w - 1)] - img[:, np.maximum(xs - 1, 0)])
    gy = 0.5 * (img[np.minimum(ys + 1, h - 1), :] - img[np.maximum(ys - 1, 0), :])
    return gx, gy


def warp(i0, i1, flow):
    """(I1x, I1y, I1w_x, I1w_y, g, rho_c) as the solver computes them before a warp's iterations."""
    h, w = i0.shape
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    gx, gy = gradient(i1)
    sx, sy = x + flow[0], y + flow[1]
    iw, wx, wy = bicubic(i1, sx, sy), bicubic(gx, sx, sy), bicubic(gy, sx, sy)
    g = wx * wx + wy * wy
    rhoc = iw - wx * flow[0] - wy * flow[1] - i0
    return gx, gy, wx, wy, g, rhoc


def divergence(px, py):
    dx = np.empty_like(px)
    dx[:, 0] = px[:, 0]
    dx[:, 1:-1] = px[:, 1:-1] - px[:, :-2]
    dx[:, -1] = -px[:, -2] if px.shape[1] > 1 else px[:, -1]
    dy = np.empty_like(py)
    dy[0] = py[0]
    dy[1:-1] = py[1:-1] - py[:-2]
    dy[-1] = -py[-2] if py.shape[0] > 1 else py[-1]
    return dx + dy


def forward_gradient(u):
    gx, gy = np.zeros_like(u), np.zeros_like(u)
    gx[:, :-1] = u[:, 1:] - u[:, :-1]
    gy[:-1] = u[1:] - u[:-1]
    return gx, gy


def iteration(wx, wy, g, rhoc, u, p):
    """One primal-dual iteration: returns (u', p', mean |u' - u|^2); u [2, H, W], p [4, H, W] (p11 p12 p21 p22)."""
    lt = LAMBDA * THETA
    rho = rhoc + (wx * u[0] + wy * u[1])
    lo, hi = rho < -lt * g, rho > lt * g
    mid = ~lo & ~hi & (g > GRAD_ZERO)
    f = np.where(mid, -rho / np.where(mid, g, 1.0), 0.0)
    d1 = np.where(lo, lt * wx, np.where(hi, -lt * wx, f * wx))
    d2 = np.where(lo, lt * wy, np.where(hi, -lt * wy, f * wy))
    un = np.stack([u[0] + d1 + THETA * divergence(p[0], p[1]), u[1] + d2 + THETA * divergence(p[2], p[3])])
    err = float(((un - u) ** 2).sum(0).mean())
    taut = TAU / THETA
    pn = np.empty_like(p)
    for c in range(2):
        gx, gy = forward_gradient(un[c])
        ng = 1.0 + taut * np.hypot(gx, gy)
        pn[2 * c] = (p[2 * c] + taut * gx) / ng
        pn[2 * c + 1] = (p[2 * c + 1] + taut * gy) / ng
    return un, pn, err


def tvl1(i0, i1):
    """Flow [2, H, W] (float64) of one pair of grey frames and the iterations [scales, WARPS] of each warp."""
    i0, i1 = np.asarray(i0, np.float64), np.asarray(i1, np.float64)
    lv = sizes(*i0.shape)
    pyr0, pyr1 = [i0], [i1]
    for hc, wc in lv[1:]:
        pyr0.append(zoom_out(pyr0[-1], hc, wc))
        pyr1.append(zoom_out(pyr1[-1], hc, wc))
    iters = np.zeros((len(lv), WARPS), np.int32)
    u = np.zeros((2,) + lv[-1])
    for s in range(len(lv) - 1, -1, -1):
        if s < len(lv) - 1:
            u = zoom_in(u, *lv[s])
        p = np.zeros((4,) + lv[s])
        for k in range(WARPS):
            _, _, wx, wy, g, rhoc = warp(pyr0[s], pyr1[s], u)
            n, err = 0, np.inf
            while err > EPSILON * EPSILON and n < MAX_ITERS:
                u, p, err = iteration(wx, wy, g, rhoc, u, p)
                n += 1
            iters[s, k] = n
    return u, iters


def texture(h, w, seed, shift=(0.0, 0.0)):
    """A seeded smooth texture in 0..255 (sum of a few sinusoids, wavelengths 10-40 px), sampled at (x - dx, y - dy):
    the flow from texture(shift=0) to texture(shift=d) is d."""
    r = np.random.RandomState(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    x, y = x - shift[0], y - shift[1]
    out = np.zeros((h, w))
    for _ in range(6):
        ang, lam, ph = r.uniform(0, np.pi), r.uniform(10, 40), r.uniform(0, 2 * np.pi)
        out += np.sin(2 * np.pi * (x * np.cos(ang) + y * np.sin(ang)) / lam + ph)
    return 128 + 100 * out / 6
