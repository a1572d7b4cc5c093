"""A second, independent restatement of the dual network (dualnet/dual.go fwd 50-103, bwd 105-132, ermahagerdmonards.go) in
numpy float64 — written from the Go sources and the four named assumptions of DESIGN.md §2 (batch-shaped BatchNorm
scale/bias, train-mode batch statistics / test-mode x/sqrt(eps), plain softmax, batch-shaped linear biases), with its own
hand-derived backward pass — used only to cross-check oracle/dual.hpp (tests/test_oracle_dual_pyref.py)."""
import numpy as np

EPS = 1e-5


def unpack(e, net):
    flat = e.net_get(net).astype(np.float64)
    nt, _ = e.param_count()
    out = []
    for i in range(nt):
        name, shape, off, size = e.param_desc(i)
        out.append((name, flat[off:off + size].reshape([s for s in shape if s > 0])))
    return out


def pack(e, tensors):
    nt, nf = e.param_count()
    flat = np.zeros(nf)
    for i in range(nt):
        _, _, off, size = e.param_desc(i)
        flat[off:off + size] = tensors[i].ravel()
    return flat


def conv(x, w):  # cross-correlation, stride 1, same padding (findPadding), no bias
    k = w.shape[2]
    p = (k - 1) // 2
    B, C, H, W = x.shape
    xp = np.pad(x, ((0, 0), (0, 0), (p, p), (p, p)))
    out = np.zeros((B, w.shape[0], H, W))
    for ky in range(k):
        for kx in range(k):
            out += np.tensordot(w[:, :, ky, kx], xp[:, :, ky:ky + H, kx:kx + W], axes=(1, 1)).transpose(1, 0, 2, 3)
    return out


def conv_bwd(x, w, dz):
    k = w.shape[2]
    p = (k - 1) // 2
    B, C, H, W = x.shape
    xp = np.pad(x, ((0, 0), (0, 0), (p, p), (p, p)))
    dw = np.zeros_like(w)
    dxp = np.zeros_like(xp)
    for ky in range(k):
        for kx in range(k):
            dw[:, :, ky, kx] = np.einsum("bohw,bchw->oc", dz, xp[:, :, ky:ky + H, kx:kx + W])
            dxp[:, :, ky:ky + H, kx:kx + W] += np.einsum("oc,bohw->bchw", w[:, :, ky, kx], dz)
    return dw, dxp[:, :, p:p + H, p:p + W]


class Unit:  # conv -> batchnorm -> rectify (m.res / the head convs)
    def __init__(self, w, gamma, beta):
        self.w, self.gamma, self.beta = w, gamma, beta

    def fwd(self, x, train):
        self.x = x
        z = conv(x, self.w)
        if train:
            mu = z.mean(axis=(0, 2, 3), keepdims=True)
            var = z.var(axis=(0, 2, 3), keepdims=True)  # biased
            self.sd = np.sqrt(var + EPS)
            self.xhat = (z - mu) / self.sd
            y = self.gamma * self.xhat + self.beta
        else:  # BatchNormOp.Reset(): stored statistics are zero; parameters: batch row 0 for every sample
            y = self.gamma[0] * (z / np.sqrt(EPS)) + self.beta[0]
        self.y = y
        return np.maximum(y, 0)

    def bwd(self, dout):
        dy = dout * (self.y > 0)
        self.dgamma, self.dbeta = dy * self.xhat, dy
        dxhat = dy * self.gamma
        m1 = dxhat.mean(axis=(0, 2, 3), keepdims=True)
        m2 = (dxhat * self.xhat).mean(axis=(0, 2, 3), keepdims=True)
        dz = (dxhat - m1 - self.xhat * m2) / self.sd
        self.dw, dx = conv_bwd(self.x, self.w, dz)
        return dx


class Net:
    def __init__(self, tensors, shared_layers):
        t = [a for _, a in tensors]
        self.L = shared_layers
        self.units = [Unit(*t[3 * i:3 * i + 3]) for i in range(1 + 2 * shared_layers)]
        o = 3 * (1 + 2 * shared_layers)
        self.pu = Unit(*t[o:o + 3]); self.pw, self.pb = t[o + 3], t[o + 4]
        self.vu = Unit(*t[o + 5:o + 8]); self.vw, self.vb, self.ow, self.ob = t[o + 8], t[o + 9], t[o + 10], t[o + 11]

    def forward(self, X, train):
        B = X.shape[0]
        cur = self.units[0].fwd(X, train)
        self.sums = []
        for i in range(self.L):
            s = self.units[1 + 2 * i].fwd(cur, train) + self.units[2 + 2 * i].fwd(cur, train)
            self.sums.append(s)
            cur = np.maximum(s, 0)
        self.tower = cur
        return self.heads(cur, train)

    def heads(self, cur, train):
        """policy logits and pre-tanh value from the tower output cur [B,K,H,W]"""
        B = cur.shape[0]
        self.ph = self.pu.fwd(cur, train).reshape(B, -1)
        self.logits = self.ph @ self.pw + (self.pb if train else self.pb[0])
        self.vh = self.vu.fwd(cur, train).reshape(B, -1)
        self.h1pre = self.vh @ self.vw + (self.vb if train else self.vb[0])
        self.h1 = np.maximum(self.h1pre, 0)
        self.vraw = (self.h1 @ self.ow + (self.ob if train else self.ob[0])).reshape(B)
        return self.logits, self.vraw

    def infer(self, X=None, tower=None):
        """softmax policy and tanh value of the planes X, or of the heads alone applied to a given tower output"""
        logits, vraw = self.forward(X, False) if tower is None else self.heads(tower, False)
        ex = np.exp(logits)
        return ex / ex.sum(axis=1, keepdims=True), np.tanh(vraw)

    def loss_grads(self, X, Pi, V):
        """cost = mean(-(Pi*logits + (1-Pi)*(1-logits))) + mean((vraw - V)^2)  (bwd, dual.go:105-132 + xent); gradients
        in Model() order."""
        B, A = Pi.shape
        logits, vraw = self.forward(X, True)
        cost = (-(Pi * logits + (1 - Pi) * (1 - logits))).mean() + ((vraw - V) ** 2).mean()
        dlog = (1 - 2 * Pi) / (B * A)
        dv = (2 * (vraw - V) / B).reshape(B, 1)
        g = {}
        g["pb"], g["pw"] = dlog, self.ph.T @ dlog
        dph = dlog @ self.pw.T
        g["ob"], g["ow"] = dv, self.h1.T @ dv
        dh1 = (dv @ self.ow.T) * (self.h1pre > 0)
        g["vb"], g["vw"] = dh1, self.vh.T @ dh1
        dvh = dh1 @ self.vw.T
        shape = self.units[0].y.shape
        dcur = self.pu.bwd(dph.reshape(B, 2, shape[2], shape[3])) + self.vu.bwd(dvh.reshape(B, 1, shape[2], shape[3]))
        for i in range(self.L - 1, -1, -1):
            ds = dcur * (self.sums[i] > 0)
            dcur = self.units[1 + 2 * i].bwd(ds) + self.units[2 + 2 * i].bwd(ds)
        self.units[0].bwd(dcur)
        out = []
        for u in self.units:
            out += [u.dw, u.dgamma, u.dbeta]
        out += [self.pu.dw, self.pu.dgamma, self.pu.dbeta, g["pw"], g["pb"], self.vu.dw, self.vu.dgamma, self.vu.dbeta,
                g["vw"], g["vb"], g["ow"], g["ob"]]
        return cost, out
