"""TEST INFRASTRUCTURE ONLY: torch-CPU emulation of the MACPO entry points of libspo (include/spo.h, spo_ma_trust.cu), a subclass
of tests/ma_emulator.py's EmulatedLib (which stays as the MAPPO-Lag tests use it) so that the host orchestration of safepo/common/ma_model.py: MACPOTrainer and of
safepo/multi_agent/macpo.py: Runner runs in the `-m "not gpu"` suite against the oracle (tests/macpo_oracle.py).  Same
positional arguments as the C functions; "pointers" are tensors.  Nothing in the package imports it; the kernels themselves
are tested on the GPU (tests/test_macpo.py)."""
import math

import torch
import torch.nn.functional as F

import ma_emulator as E
from ma_emulator import _mem

LOG_SQRT_2PI = E.LOG_SQRT_2PI
WORK_FLOATS = 256 * 4 + 4


def logstd_curvature(log_std, x_coef, y_coef):
    """d^2 KL_j / d log_std_j^2 at new = old for MACPO's KL (macpo.py:163-164, with its 1e-8), closed form in float64 -- the
    formula spo_ma_fvp_finalize evaluates."""
    ls = log_std.double()
    sg = torch.sigmoid(ls / x_coef)
    s = y_coef * sg
    s0 = s * s
    D = 1e-8 + 2.0 * s0
    f1 = -1.0 / s - 4.0 * s * s0 / D ** 2
    f2 = 1.0 / s0 - 4.0 * s0 / D ** 2 + 32.0 * s0 * s0 / D ** 3
    d1 = y_coef * sg * (1 - sg) / x_coef
    d2 = y_coef * sg * (1 - sg) * (1 - 2 * sg) / x_coef ** 2
    return f2 * d1 * d1 + f1 * d2


def _std(log_std, x, y):
    return torch.sigmoid(log_std / x) * y


def _layer_shape(K, H):
    """The shape checks of the C functions (spo_ma.cu / spo_ma_trust.cu): a shape the kernels reject fails here too."""
    if not (K >= 2 and K % 2 == 0 and 128 <= H <= 512 and H % 128 == 0):
        raise AssertionError(f"K={K}, H={H}: the C function returns SPO_ERR_UNSUPPORTED")


def _act_shape(A):
    if not 1 <= A <= 32:
        raise AssertionError(f"act_dim={A}: the C function returns SPO_ERR_UNSUPPORTED")


class EmulatedMACPOLib(E.EmulatedLib):
    """EmulatedLib plus the MACPO entry points, with the C functions' shape checks on the layer and head entry points."""

    def spo_ma_work_floats(self):
        return WORK_FLOATS

    def spo_ma_mlp_layer(self, x, n, K, W, b, lnw, lnb, H, *rest):
        _layer_shape(K, H)
        return super().spo_ma_mlp_layer(x, n, K, W, b, lnw, lnb, H, *rest)

    def spo_ma_mlp_layer_train(self, x, n, K, W, b, lnw, lnb, H, *rest):
        _layer_shape(K, H)
        return super().spo_ma_mlp_layer_train(x, n, K, W, b, lnw, lnb, H, *rest)

    def spo_ma_mlp_layer_jvp(self, x, dx, n, K, W, dW, db, pre, lnw, dlnw, dlnb, H, linw, linb, dlinw, dlinb, dout, stream):
        _layer_shape(K, H)
        x = _mem(x, n, K)
        if linw is not None:
            m = x.mean(-1, keepdim=True)
            xh = (x - m) * torch.rsqrt(((x - m) ** 2).mean(-1, keepdim=True) + 1e-5)
            xin, dxin = xh * _mem(linw, K) + _mem(linb, K), xh * _mem(dlinw, K) + _mem(dlinb, K)
        else:
            xin, dxin = x, _mem(dx, n, K)
        dz = dxin @ _mem(W, H, K).t() + xin @ _mem(dW, H, K).t() + _mem(db, H)
        h = _mem(pre, n, H)
        dh = dz * torch.where(h > 0, torch.ones_like(h), h + 1)
        m = h.mean(-1, keepdim=True)
        rstd = torch.rsqrt(((h - m) ** 2).mean(-1, keepdim=True) + 1e-5)
        hn = (h - m) * rstd
        dhn = rstd * (dh - dh.mean(-1, keepdim=True) - hn * (dh * hn).mean(-1, keepdim=True))
        _mem(dout, n, H).copy_(_mem(lnw, H) * dhn + _mem(dlnw, H) * hn + _mem(dlnb, H))
        return 0

    def spo_ma_head_jvp(self, feat, dfeat, n, H, W, dW, db, A, log_std, x_coef, y_coef, dmean, part, stream):
        _act_shape(A)
        sd = _std(_mem(log_std, A), x_coef, y_coef)
        w = 2.0 / (1e-8 + 2 * sd * sd) / n
        dm = w * (_mem(dfeat, n, H) @ _mem(W, A, H).t() + _mem(feat, n, H) @ _mem(dW, A, H).t() + _mem(db, A))
        _mem(dmean, n, A).copy_(dm)
        nb = (n + 31) // 32
        p = _mem(part, nb, A)
        for blk in range(nb):
            p[blk] = dm[32 * blk:32 * blk + 32].sum(0)
        return 0

    def spo_ma_fvp_finalize(self, gn, v, out, P, log_std, off, A, x_coef, y_coef, damping, stream):
        g, v, o = _mem(gn, P), _mem(v, P), _mem(out, P)
        f = g.clone()
        f[off:off + A] = (logstd_curvature(_mem(log_std, A), x_coef, y_coef) * v[off:off + A].double()).float()
        o.copy_(f + damping * v)
        return 0

    def spo_ma_ratio_loss(self, mean, n, log_std, A, actions, old_logp, adv, factor, sign, x_coef, y_coef, dmean, part, stream):
        _act_shape(A)
        mu, ls = _mem(mean, n, A), _mem(log_std, A)
        sd = _std(ls, x_coef, y_coef)
        diff = _mem(actions, n, A) - mu
        lp = -(diff ** 2) / (2 * sd ** 2) - sd.log() - LOG_SQRT_2PI
        ratio = torch.exp(lp - _mem(old_logp, n, A)).prod(-1)
        term = ratio * _mem(factor, n) * _mem(adv, n)
        c = sign * term / n
        dm = c[:, None] * diff / sd ** 2
        sg = torch.sigmoid(ls / x_coef)
        ds = c[:, None] * (diff ** 2 / sd ** 3 - 1 / sd) * (y_coef * sg * (1 - sg) / x_coef)
        _mem(dmean, n, A).copy_(dm)
        nb = (n + 31) // 32
        p = _mem(part, nb, 3, A)
        p.zero_()
        for blk in range(nb):
            r = slice(32 * blk, min(n, 32 * blk + 32))
            p[blk, 0, 0] = term[r].sum()
            p[blk, 1], p[blk, 2] = dm[r].sum(0), ds[r].sum(0)
        return 0

    def spo_ma_dots(self, a0, b0, a1, b1, a2, b2, a3, b3, ndot, P, work, out, stream):
        o = _mem(out, ndot)
        for s, (a, b) in enumerate(((a0, b0), (a1, b1), (a2, b2), (a3, b3))[:ndot]):
            o[s] = torch.dot(_mem(a, P), _mem(b, P))
        return 0

    def spo_ma_cg_begin(self, b, x, r, p, P, work, state, stream):
        b = _mem(b, P)
        _mem(x, P).zero_()
        _mem(r, P).copy_(b)
        _mem(p, P).copy_(b)
        st = _mem(state, 4)
        st.zero_()
        st[0] = torch.dot(b, b)
        return 0

    def spo_ma_cg_update(self, x, r, p, Ap, P, tol, work, state, stream):
        st = _mem(state, 4)
        if st[3] != 0:
            return 0
        x, r, p, Ap = _mem(x, P), _mem(r, P), _mem(p, P), _mem(Ap, P)
        rdotr = st[0].clone()
        alpha = rdotr / (st[1] + 1e-8)
        x += alpha * p
        r -= alpha * Ap
        new = torch.dot(r, r)
        beta = new / rdotr
        p.copy_(r + beta * p)
        st[0], st[2] = new, beta
        if new < tol:
            st[3] = 1.0
        return 0

    def spo_ma_step_dir(self, xg, xb, c, nu, use_a, x, P, stream):
        xb = _mem(xb, P)
        _mem(x, P).copy_(c * (_mem(xg, P) + nu * xb) if use_a else nu * xb)
        return 0

    def spo_ma_ls_trial(self, old, x, xsq, coef, out, P, stream):
        x = _mem(x, P)
        nrm = torch.sqrt(_mem(xsq, 1)[0])
        if nrm > 0.5:
            x.copy_(x * 0.5 / nrm)
        _mem(out, P).copy_(_mem(old, P) - coef * x)
        return 0

    def spo_ma_linesearch_eval(self, mean_new, mean_old, ls_new, ls_old, A, actions, old_logp, adv, cost_adv, factor, n, x_coef, y_coef, work, out,
                               stream):
        mn, mo = _mem(mean_new, n, A), _mem(mean_old, n, A)
        sn, so = _std(_mem(ls_new, A), x_coef, y_coef).expand(n, A), _std(_mem(ls_old, A), x_coef, y_coef).expand(n, A)
        lp = torch.distributions.Normal(mn, sn).log_prob(_mem(actions, n, A))
        ratio = torch.prod(torch.exp(lp - _mem(old_logp, n, A)), dim=-1, keepdim=True)
        f = _mem(factor, n, 1)
        kl = (torch.log(so) - torch.log(sn) + (so.pow(2) + (mo - mn).pow(2)) / (1e-8 + 2.0 * sn.pow(2)) - 0.5).sum(1, keepdim=True)
        o = _mem(out, 4)
        o[0] = -torch.sum(ratio * f * _mem(adv, n, 1), dim=-1, keepdim=True).mean()
        o[1] = torch.sum(ratio * f * _mem(cost_adv, n, 1), dim=-1, keepdim=True).mean()
        o[2] = kl.mean()
        o[3] = ratio.mean()
        return 0


def install(monkeypatch):
    """ma_emulator.install with the MACPO entry points."""
    lib = E.install(monkeypatch)
    from safepo import _lib as L
    mlib = EmulatedMACPOLib()
    monkeypatch.setattr(L, "lib", lambda: mlib)
    return mlib
