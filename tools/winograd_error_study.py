#!/usr/bin/env python
"""Feasibility arithmetic for DESIGN.md §10: error of a Winograd F(2x2,3x3) formulation of one tower layer when its 16
element-wise GEMMs run as fp16 hi/lo 3-pass products with fp32 accumulation (what the fp16 tensor cores give), against the
direct 9-tap form with the same split — both measured against an fp64 convolution.  CPU only (numpy), one layer,
C = 256, 19x19, a few boards; activations are ReLU outputs, filters GlorotU like the reference's init."""
import numpy as np

rng = np.random.default_rng(0)
C, H, W, NB = 256, 19, 19, 2


def split(x):
    """x (fp32) -> fp16 hi + fp16 lo at a power-of-two scale that puts absmax in [2^13, 2^14)."""
    m = np.abs(x).max()
    e = 13 - int(np.floor(np.log2(m)))
    xs = (x * np.float32(2.0 ** e)).astype(np.float32)
    hi = xs.astype(np.float16)
    lo = (xs - hi.astype(np.float32)).astype(np.float16)
    return hi.astype(np.float32), lo.astype(np.float32), e


PASSES = 3


def mm3(a, b):
    """PASSES-pass product of split operands, fp32 accumulate: a [M,K], b [K,N] (3: hi*hi + hi*lo + lo*hi; 2: drops lo*hi)."""
    ah, al, ea = split(a)
    bh, bl, eb = split(b)
    acc = ah @ bh + ah @ bl
    if PASSES >= 3:
        acc = acc + al @ bh
    return acc * np.float32(2.0 ** -(ea + eb))


x = np.maximum(rng.normal(0, 1, (NB, C, H, W)), 0).astype(np.float32)
lim = np.sqrt(6.0 / ((C + C) * 9))
w = rng.uniform(-lim, lim, (C, C, 3, 3)).astype(np.float32)

# fp64 reference (cross-correlation, same padding)
xp = np.pad(x.astype(np.float64), ((0, 0), (0, 0), (1, 1), (1, 1)))
ref = np.zeros((NB, C, H, W))
for ky in range(3):
    for kx in range(3):
        ref += np.einsum("oc,nchw->nohw", w[:, :, ky, kx].astype(np.float64), xp[:, :, ky:ky + H, kx:kx + W])

# direct form, split (one GEMM with K = 9*C)
for PASSES in (3, 2):
    xp32 = np.pad(x, ((0, 0), (0, 0), (1, 1), (1, 1)))
    cols = np.stack([xp32[:, :, ky:ky + H, kx:kx + W] for ky in range(3) for kx in range(3)], axis=1)  # [N,9,C,H,W]
    A = cols.transpose(0, 3, 4, 1, 2).reshape(NB * H * W, 9 * C)
    Bm = w.transpose(2, 3, 1, 0).reshape(9 * C, C)
    direct = mm3(A, Bm).reshape(NB, H, W, C).transpose(0, 3, 1, 2)

    # Winograd F(2x2,3x3)
    Bt = np.array([[1, 0, -1, 0], [0, 1, 1, 0], [0, -1, 1, 0], [0, 1, 0, -1]], np.float32)
    G = np.array([[1, 0, 0], [.5, .5, .5], [.5, -.5, .5], [0, 0, 1]], np.float32)
    At = np.array([[1, 1, 1, 0], [0, 1, -1, -1]], np.float32)
    TH = (H + 1) // 2  # 10 x 10 tiles of 2x2 outputs over a 20x20 padded output
    xpw = np.pad(x, ((0, 0), (0, 0), (1, 2), (1, 2)))  # input 22x22
    U = np.einsum("ij,ocjk,lk->iloc", G, w, G).astype(np.float32)  # [4,4,Co,Ci]
    tiles = np.stack([xpw[:, :, 2 * ty:2 * ty + 4, 2 * tx:2 * tx + 4] for ty in range(TH) for tx in range(TH)], axis=1)  # [N,T,C,4,4]
    V = np.einsum("ij,ntcjk,lk->ilntc", Bt, tiles, Bt).astype(np.float32)  # [4,4,N,T,C]
    M = np.zeros((4, 4, NB * TH * TH, C), np.float32)
    for i in range(4):
        for j in range(4):
            M[i, j] = mm3(V[i, j].reshape(NB * TH * TH, C), U[i, j].T)
    Y = np.einsum("ij,jkto,lk->tilo", At, M, At)  # [T*,2,2,Co]
    Y = Y.reshape(NB, TH, TH, 2, 2, C).transpose(0, 5, 1, 3, 2, 4).reshape(NB, C, 2 * TH, 2 * TH)[:, :, :H, :W]

    scale = np.abs(ref).max()
    rms = np.sqrt((ref ** 2).mean())
    for name, y in (("direct 9-tap, %d-pass split" % PASSES, direct), ("Winograd F(2x2,3x3), %d-pass split" % PASSES, Y)):
        err = np.abs(y - ref)
        print("%-36s max|err| %.3e  rms err %.3e   (output max %.3g, rms %.3g)  max|err|/rms(out) %.2e" %
              (name, err.max(), np.sqrt((err ** 2).mean()), scale, rms, err.max() / rms))
# plain fp32 (what the oracle / fp32 tower computes) for reference
A = cols.transpose(0, 3, 4, 1, 2).reshape(NB * H * W, 9 * C)
fp32 = (A @ Bm).reshape(NB, H, W, C).transpose(0, 3, 1, 2)
err = np.abs(fp32 - ref)
print("%-36s max|err| %.3e  rms err %.3e" % ("fp32 GEMM (numpy)", err.max(), np.sqrt((err ** 2).mean())))
