"""TEST INFRASTRUCTURE ONLY: tests/ma_emulator.py's torch-CPU emulation of libspo extended by the MAPPO / HAPPO loss heads
(spo_ma_ppo_actor_loss, spo_ma_ppo_actor_finalize, spo_ma_value_loss_masked), so that the host orchestration of
MAPPOTrainer / HAPPOTrainer and their runners runs in the `-m "not gpu"` suite against the oracle.  Same positional
arguments as the C functions; "pointers" are the tensors themselves.  The kernels are tested on the GPU
(tests/test_mappo_happo.py)."""
import torch

from ma_emulator import LOG_SQRT_2PI, EmulatedLib, _mem


class PPOEmulatedLib(EmulatedLib):
    def spo_ma_ppo_actor_loss(self, feat, n, H, W, b, log_std, A, actions, old_logp, adv, cost_adv, lamda, factor, masks, mask_sum,
                              ratio_mode, clip_lo, clip_hi, x_coef, y_coef, dmean, imp, part, stream):
        mu = _mem(feat, n, H) @ _mem(W, A, H).t() + _mem(b, A)
        std = torch.sigmoid(_mem(log_std, A) / x_coef) * y_coef
        diff = _mem(actions, n, A) - mu
        lp = -(diff ** 2) / (2 * std ** 2) - std.log() - LOG_SQRT_2PI
        ratio = torch.exp(lp - _mem(old_logp, n, A))
        a_h = _mem(adv, n) if cost_adv is None else _mem(adv, n) - _mem(lamda, 1) * _mem(cost_adv, n)
        fac = torch.ones(n) if factor is None else _mem(factor, n)
        m = torch.ones(n) if masks is None else _mem(masks, n)
        w = torch.full((n,), 1.0 / n) if masks is None else m / _mem(mask_sum, 1)
        w_ = ratio.prod(-1, keepdim=True) if ratio_mode == 0 else ratio           # [n, 1] or [n, A]
        s1, s2 = w_ * a_h[:, None], w_.clamp(clip_lo, clip_hi) * a_h[:, None]
        crow = torch.where(s1 <= s2, (-fac * a_h * w)[:, None], torch.zeros_like(s1)) * w_
        dm = crow * diff / std ** 2
        ds = crow * (diff ** 2 / std ** 3 - 1 / std)
        _mem(dmean, n, A).copy_(dm)
        _mem(imp, n * w_.shape[1]).copy_(w_.reshape(-1))
        loss_row = -fac * torch.min(s1, s2).sum(-1) * (1.0 if masks is None else m)
        nb = (n + 31) // 32
        p = _mem(part, nb, 66)
        p.zero_()
        for blk in range(nb):
            r = slice(32 * blk, min(n, 32 * blk + 32))
            p[blk, 0], p[blk, 1] = loss_row[r].sum(), w_[r].sum()
            p[blk, 2:2 + A] = dm[r].sum(0)
            p[blk, 34:34 + A] = ds[r].sum(0)
        return 0

    def spo_ma_ppo_actor_finalize(self, part, nblk, n, mask_sum, ratio_mode, log_std, A, x_coef, y_coef, entropy_coef, g_b, g_log_std,
                                  scalars, stream):
        tot = _mem(part, nblk, 66).sum(0)
        sg = torch.sigmoid(_mem(log_std, A) / x_coef)
        std = sg * y_coef
        e = 0.5 + LOG_SQRT_2PI + std.log()
        if mask_sum is None:
            coef, ent, den = entropy_coef / (A * std), e.mean(), n
        else:
            ms = _mem(mask_sum, 1)[0]
            q = ms / ms
            coef, ent, den = q * entropy_coef / std, q * e.sum(), ms
        _mem(g_log_std, A).copy_((tot[34:34 + A] - coef) * (y_coef * sg * (1 - sg) / x_coef))
        _mem(g_b, A).copy_(tot[2:2 + A])
        sc = _mem(scalars, 3)
        sc[0], sc[1], sc[2] = tot[0] / den, ent, tot[1] / (n * A if ratio_mode == 1 else n)
        return 0

    def spo_ma_value_loss_masked(self, v, vp, rn_c, rn_o, masks, mask_sum, n, clip, delta, coef, dv, part, stream):
        w = _mem(masks, n) / _mem(mask_sum, 1)
        tmp = torch.empty(((n + 255) // 256) * 2)
        self.spo_ma_value_loss(v, vp, rn_c, rn_o, n, clip, delta, 1.0, dv, tmp, stream)
        g = _mem(dv, n)
        g.mul_(coef * w)
        # the unweighted rows' losses, recomputed to weight them
        vv, vvp, rc, ro = _mem(v, n), _mem(vp, n), _mem(rn_c, n), _mem(rn_o, n)
        ec, eo = rc - (vvp + (vv - vvp).clamp(-clip, clip)), ro - vv

        def hub(e):
            return (e.abs() <= delta).float() * e ** 2 / 2 + (e > delta).float() * delta * (e.abs() - delta / 2)
        L = torch.max(hub(eo), hub(ec)) * w
        nb = (n + 255) // 256
        p = _mem(part, nb, 2)
        for blk in range(nb):
            r = slice(256 * blk, min(n, 256 * blk + 256))
            p[blk, 0], p[blk, 1] = L[r].sum(), g[r].sum()
        return 0


def install(monkeypatch):
    """Route the package's library calls to this emulation for one test (pytest's monkeypatch undoes it)."""
    import ma_emulator
    from safepo import _lib as L
    ma_emulator.install(monkeypatch)
    lib = PPOEmulatedLib()
    monkeypatch.setattr(L, "lib", lambda: lib)
    return lib
