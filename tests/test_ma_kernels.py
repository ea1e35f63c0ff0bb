"""The multi-agent kernels (csrc/spo_ma.cu, spo_ma_update.cu, spo_ma_trust.cu) per entry point and per tensor against float64.

The float64 reference below restates the reference's forward formulas with the dtype as a parameter -- the
[Linear -> ELU -> LayerNorm] block, the DiagGaussian and value heads, the clipped surrogate on the product of ratios, the
clipped one-sided-Huber value loss with torch.max, PopArt, the Lagrange step, clip_grad_norm_ + Adam, MACPO's KL and its
Fisher-vector product -- and takes every derivative by autograd.  It does not restate any hand-derived derivative of the
kernels (tests/ma_emulator.py and tests/macpo_emulator.py do), so a formula mistake shared by a kernel and its emulator
cannot pass here.  In float32 it equals oracle/ma_oracle.py's OracleMATrainer.ppo_update and tests/macpo_oracle.py bit for
bit (the CPU tests), so it has the semantics the golden fixtures pin.

The GPU tests call each C-ABI entry point with float32 inputs and compare every output with float64 computed from the same
inputs, at the shapes and branch edges where the kernels could go wrong: H = 384, K = 2, n = 1, act_dim 1 and 32, every
clip / Huber / ReLU branch, a CG stop.  Branch decisions are built with a margin or exactly on the boundary, and the tests
assert how many rows fall in each branch.  Then whole MultiAgentTrainer.ppo_update / MACPOTrainer steps are read out per
tensor at shapes no other test runs.  Run with ``-s`` to see the measured maxima."""
import math

import pytest
import torch
import torch.nn.functional as F
from torch.distributions import Normal

from oracle import ma_oracle as MA

# Bars: error / scale of the quantity (the tensor's max |float64|, or the named scale), each at most 4x the largest error
# measured over this file's matrix on one H100 80GB HBM3 (in brackets).  The whole-step readouts go through three fp32
# layers and their LayerNorms; the kernels on their own stay at a few 1e-6.
BAR = dict(
    layer=4e-6,           # [1.2e-6] out, pre, xn of spo_ma_mlp_layer(_train)
    head=1.2e-5,          # [3.1e-6] actions, per-dimension log-probs, values
    ln_bwd=9e-6,          # [2.4e-6] dz and the column sums of spo_ma_ln_elu_bwd / spo_ma_ln_in_bwd
    actor=3e-5,           # [8.3e-6] dmean, importance weights, g_b, g_log_std
    actor_loss=1.2e-5,    # [3.2e-6] policy loss (relative to the mean |term|), entropy
    value=2.4e-7,         # [6.2e-8] dv, its sum and the loss
    popart=9e-7,          # [2.3e-7] state; outputs relative to max |x| / sd
    lagrange=3e-7,        # [8.5e-8] lambda, relative to |lambda - delta rate| + lambda
    adam=1.4e-5,          # [3.6e-6] norm, clip coefficient, weight movement, m, v
    gemm=8e-6,            # [2.0e-6] sliced A^T B
    jvp=1e-5,             # [2.8e-6] layer tangent
    head_jvp=1.2e-6,      # [3.4e-7] weighted mean tangent and its column sums
    ratio=8e-6,           # [2.2e-6] ratio loss, dmean, g_b, g_log_std
    finalize=4e-7,        # [1.2e-7] FVP finalize, whole vector and log_std block
    ls_loss=9e-6,         # [2.5e-6] line-search losses (relative to the mean |term|) and mean ratio
    ls_kl=1.2e-6,         # [3.1e-7] line-search KL, relative to the size of its A terms
    vec=2.8e-7,           # [7.4e-8] dots, CG step, step direction, trial weights
    step_grad=7e-5,       # [1.8e-5] MultiAgentTrainer.ppo_update: every tensor's gradient before the clip
    step_scalar=1.5e-4,   # [3.8e-5] ... its eight returned values, lambda, PopArt state
    step_fvp=5e-5,        # [1.3e-5] MACPOTrainer.fvp per tensor
    step_surr=6e-5)       # [1.7e-5] MACPOTrainer.surrogate_grad per tensor and the surrogate
MEASURED = {}

X_COEF, Y_COEF = 1.7, 0.4          # std = sigmoid(log_std / x) * y with x != 1


# ======================================================= float64 reference =======================================================
def ln(x, w, b):
    return F.layer_norm(x, (x.shape[-1],), w, b)


def block(x, W, b, lw, lb, lin=None):
    """MLPLayer's [Linear -> ELU -> LayerNorm] (mlp.py:18-27), with MLPBase's input LayerNorm first when ``lin`` = (w, b)."""
    if lin is not None:
        x = ln(x, *lin)
    return ln(F.elu(F.linear(x, W, b)), lw, lb)


def features(p, x, layer_N):
    """MLPBase.forward (mlp.py:56-61)."""
    x = ln(x, p["base.feature_norm.weight"], p["base.feature_norm.bias"])
    x = ln(F.elu(F.linear(x, p["base.mlp.fc1.0.weight"], p["base.mlp.fc1.0.bias"])), p["base.mlp.fc1.2.weight"], p["base.mlp.fc1.2.bias"])
    for i in range(layer_N):
        x = ln(F.elu(F.linear(x, p[f"base.mlp.fc2.{i}.0.weight"], p[f"base.mlp.fc2.{i}.0.bias"])), p[f"base.mlp.fc2.{i}.2.weight"],
               p[f"base.mlp.fc2.{i}.2.bias"])
    return x


def diag_gaussian(mean, log_std, x_coef, y_coef):
    """DiagGaussian (distributions.py:38-42): std = sigmoid(log_std / x) * y."""
    return Normal(mean, torch.sigmoid(log_std / x_coef) * y_coef)


def actor_dist(p, obs, layer_N, x_coef, y_coef):
    feat = features(p, obs, layer_N)
    return diag_gaussian(F.linear(feat, p["act.action_out.fc_mean.weight"], p["act.action_out.fc_mean.bias"]), p["act.action_out.log_std"],
                         x_coef, y_coef)


def critic_value(p, x, layer_N):
    return F.linear(features(p, x, layer_N), p["v_out.weight"], p["v_out.bias"])


def surrogate(log_probs, old_log_probs, adv_targ, cost_adv_targ, factor, lamda, clip):
    """mappolag.py:160-166: clipped surrogate on the product of the per-dimension ratios with the lambda-mixed advantage."""
    adv = adv_targ - lamda * cost_adv_targ
    imp = torch.prod(torch.exp(log_probs - old_log_probs), dim=-1, keepdim=True)
    surr1 = imp * adv
    surr2 = torch.clamp(imp, 1.0 - clip, 1.0 + clip) * adv
    return -torch.sum(factor * torch.min(surr1, surr2), dim=-1, keepdim=True).mean(), imp


def huber(e, d):
    """util.py:19-22: quadratic for |e| <= d, linear for e > d, zero for e < -d (sic)."""
    a = (abs(e) <= d).to(e.dtype)
    b = (e > d).to(e.dtype)
    return a * e ** 2 / 2 + b * d * (abs(e) - d / 2)


def value_loss(values, value_preds, ret_c, ret_o, clip, delta):
    """cal_value_loss (mappolag.py:121-133) with the two normalised returns given."""
    vpc = value_preds + (values - value_preds).clamp(-clip, clip)
    return torch.max(huber(ret_o - values, delta), huber(ret_c - vpc, delta)).mean()


class PopArt:
    """PopArt(1).forward / running_mean_var (popart.py:64-112) in ``dtype``."""

    def __init__(self, dtype, beta=0.99999, epsilon=1e-5):
        self.beta, self.epsilon = beta, epsilon
        self.running_mean = torch.zeros(1, dtype=dtype)
        self.running_mean_sq = torch.zeros(1, dtype=dtype)
        self.debiasing_term = torch.tensor(0.0, dtype=dtype)
        self.dtype = dtype

    def state(self):
        return torch.stack([self.running_mean[0], self.running_mean_sq[0], self.debiasing_term])

    def normalize(self, x):
        x = x.to(self.dtype)
        d = x.detach()
        batch_mean, batch_sq_mean = d.mean(dim=(0,)), (d ** 2).mean(dim=(0,))
        weight = self.beta
        self.running_mean.mul_(weight).add_(batch_mean * (1.0 - weight))
        self.running_mean_sq.mul_(weight).add_(batch_sq_mean * (1.0 - weight))
        self.debiasing_term.mul_(weight).add_(1.0 * (1.0 - weight))
        mean = self.running_mean / self.debiasing_term.clamp(min=self.epsilon)
        mean_sq = self.running_mean_sq / self.debiasing_term.clamp(min=self.epsilon)
        var = (mean_sq - mean ** 2).clamp(min=1e-2)
        return (x - mean[None]) / torch.sqrt(var)[None]


def lagrange_step(lamda, imp, cost_adv_targ, aver_episode_costs, cost_limit, gamma, rate):
    """mappolag.py:169-172."""
    delta = -((aver_episode_costs.mean() - cost_limit) * (1 - gamma) + (imp * cost_adv_targ)).mean().detach()
    return torch.nn.ReLU()(lamda - (delta * rate))


def clip_adam(params, lr, eps, weight_decay, max_grad_norm, state=None):
    """clip_grad_norm_ then one torch.optim.Adam step on ``params`` (leaves with .grad); ``state``: per-param (step, m, v) to
    resume from.  Returns the total norm and the optimiser."""
    opt = torch.optim.Adam(params, lr=lr, eps=eps, weight_decay=weight_decay, foreach=False)
    if state is not None:
        for p, (step, m, v) in zip(params, state):
            opt.state[p] = dict(step=torch.tensor(float(step)), exp_avg=m.clone(), exp_avg_sq=v.clone())
    norm = torch.nn.utils.clip_grad_norm_(params, max_grad_norm)
    opt.step()
    return norm, opt


def ref_ppo_update(states, s, cfg, dtype, layer_N, popart=None):
    """MAPPO_L_Trainer.ppo_update (mappolag.py:135-199) on copies of ``states`` (actor, critic, cost critic) in ``dtype``.
    Returns the parameter leaves (after the step; .grad clipped), the gradients before the clip, the eight returned values,
    the new lambda and the PopArt normaliser."""
    c = cfg
    nets = [{k: v.detach().to(dtype).clone().requires_grad_(True) for k, v in st.items()} for st in states]
    s = {k: torch.as_tensor(v).to(dtype) for k, v in s.items()}
    popart = PopArt(dtype) if popart is None else popart
    actor, critic, cost_critic = nets
    x, y = c["std_x_coef"], c["std_y_coef"]
    dist = actor_dist(actor, s["obs"], layer_N, x, y)
    action_log_probs = dist.log_prob(s["actions"])
    dist_entropy = dist.entropy().mean()
    values = critic_value(critic, s["share_obs"], layer_N)
    cost_values = critic_value(cost_critic, s["share_obs"], layer_N)
    policy_loss, imp = surrogate(action_log_probs, s["old_action_log_probs"], s["adv_targ"], s["cost_adv_targ"], s["factor"],
                                 c["lamda_lagr"], c["clip_param"])
    pre_clip, norms = [], []

    def step(net, loss, lr):
        params = list(net.values())
        for p in params:
            p.grad = None
        loss.backward()
        pre_clip.append({k: p.grad.detach().clone() for k, p in net.items()})
        norms.append(clip_adam(params, lr, c["opti_eps"], c["weight_decay"], c["max_grad_norm"])[0])

    step(actor, policy_loss - dist_entropy * c["entropy_coef"], c["actor_lr"])
    lamda = lagrange_step(c["lamda_lagr"], imp.detach(), s["cost_adv_targ"], s["aver_episode_costs"], c["cost_limit"], c["gamma"],
                          c["lagrangian_coef_rate"])

    def cal_value_loss(v, vp, ret):
        ret_c = popart.normalize(ret)          # PopArt.forward updates the statistics, then normalises -- twice
        ret_o = popart.normalize(ret)
        return value_loss(v, vp, ret_c, ret_o, c["clip_param"], c["huber_delta"])

    vl = cal_value_loss(values, s["value_preds"], s["returns"])
    step(critic, vl * c["value_loss_coef"], c["critic_lr"])
    cl = cal_value_loss(cost_values, s["cost_preds"], s["cost_returns"])
    step(cost_critic, cl * c["value_loss_coef"], c["critic_lr"])
    out = dict(value_loss=vl.detach(), critic_grad_norm=norms[1], policy_loss=policy_loss.detach(), dist_entropy=dist_entropy.detach(),
               actor_grad_norm=norms[0], imp_weights=imp.detach(), cost_loss=cl.detach(), cost_grad_norm=norms[2])
    return dict(nets=nets, grads=pre_clip, out=out, lamda=lamda, popart=popart, imp=imp.detach(), log_probs=action_log_probs.detach())


def kl_terms(mu, std, mu_old, std_old):
    """MACPO_Trainer.kl_divergence (macpo.py:153-166) per row: its log terms and its 1e-8 as the reference has them."""
    logstd = torch.log(std)
    mu_old, std_old = mu_old.detach(), std_old.detach()
    logstd_old = torch.log(std_old)
    kl = logstd_old - logstd + (std_old.pow(2) + (mu_old - mu).pow(2)) / (1e-8 + 2.0 * std.pow(2)) - 0.5
    return kl.sum(1, keepdim=True)


def ref_fvp(p, obs, v, layer_N, x_coef, y_coef, damping=0.1):
    """macpo.py:187-198: double backprop of the mean KL of the actor against itself, plus damping * v (v in state_dict order)."""
    params = list(p.values())
    new = actor_dist(p, obs, layer_N, x_coef, y_coef)
    old = actor_dist(p, obs, layer_N, x_coef, y_coef)
    kl = kl_terms(new.mean, new.stddev, old.mean, old.stddev).mean()
    g = torch.cat([t.view(-1) for t in torch.autograd.grad(kl, params, create_graph=True)])
    hp = torch.autograd.grad((g * v).sum(), params)
    return torch.cat([t.contiguous().view(-1) for t in hp]).data + damping * v


def ratio_surrogates(log_probs, old_log_probs, factor, adv, cost_adv):
    """macpo.py:239-251: (reward loss, cost loss, ratio)."""
    ratio = torch.prod(torch.exp(log_probs - old_log_probs), dim=-1, keepdim=True)
    return (-torch.sum(ratio * factor * adv, dim=-1, keepdim=True).mean(), torch.sum(ratio * factor * cost_adv, dim=-1, keepdim=True).mean(),
            ratio)


def linesearch_quantities(new, old, actions, old_log_probs, factor, adv, cost_adv):
    """macpo.py:349-368 for two DiagGaussians: (new reward loss, new cost loss, mean KL(old || new), mean ratio)."""
    rl, cl, ratio = ratio_surrogates(new.log_prob(actions), old_log_probs, factor, adv, cost_adv)
    return rl, cl, kl_terms(new.mean, new.stddev, old.mean, old.stddev).mean(), ratio.mean()


# ============================================================ helpers ============================================================
def _state(g, din, H, A, head, layer_N=2):
    """A MultiAgentActor / MultiAgentCritic state dict (reference names) with non-trivial LayerNorm parameters and biases."""
    st = {"base.feature_norm.weight": 1 + 0.1 * torch.randn(din, generator=g), "base.feature_norm.bias": 0.1 * torch.randn(din, generator=g)}
    names = ["fc1"] + [f"fc2.{i}" for i in range(layer_N)]
    for li, name in enumerate(names):
        k = din if li == 0 else H
        st[f"base.mlp.{name}.0.weight"] = torch.randn(H, k, generator=g) * (1.4 / k ** 0.5)
        st[f"base.mlp.{name}.0.bias"] = 0.1 * torch.randn(H, generator=g)
        st[f"base.mlp.{name}.2.weight"] = 1 + 0.1 * torch.randn(H, generator=g)
        st[f"base.mlp.{name}.2.bias"] = 0.1 * torch.randn(H, generator=g)
    if head == "actor":
        st["act.action_out.log_std"] = torch.ones(A) + 0.3 * torch.randn(A, generator=g)
        st["act.action_out.fc_mean.weight"] = torch.randn(A, H, generator=g) * 0.05
        st["act.action_out.fc_mean.bias"] = 0.1 * torch.randn(A, generator=g)
    else:
        st["v_out.weight"] = torch.randn(1, H, generator=g) * 0.1
        st["v_out.bias"] = 0.1 * torch.randn(1, generator=g)
    return st


def _sample(g, N, D, DS, A, oa_state, layer_N, x_coef, y_coef, ret_scale=4.0):
    with torch.no_grad():
        p = {k: v.float() for k, v in oa_state.items()}
        obs, share = torch.randn(N, D, generator=g) * 2 + 0.5, torch.randn(N, DS, generator=g) * 3
        dist = actor_dist(p, obs, layer_N, x_coef, y_coef)
        actions = dist.mean + dist.stddev * torch.randn(N, A, generator=g)
        logp = dist.log_prob(actions)
    return dict(share_obs=share, obs=obs, actions=actions, value_preds=0.3 * torch.randn(N, 1, generator=g),
                returns=torch.randn(N, 1, generator=g) * ret_scale + 1, old_action_log_probs=logp + 0.05 * torch.randn(N, A, generator=g) / A ** 0.5,
                adv_targ=torch.randn(N, 1, generator=g), factor=torch.rand(N, 1, generator=g) + 0.5,
                cost_preds=0.3 * torch.randn(N, 1, generator=g), cost_returns=torch.randn(N, 1, generator=g).abs() * 30,
                cost_adv_targ=torch.randn(N, 1, generator=g), aver_episode_costs=torch.rand(N, 1, generator=g) * 60)


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


def _call(name, *args):
    from safepo import _lib as L
    L.check(getattr(L.lib(), name)(*args), name)


def _ptr(t):
    from safepo import _lib as L
    return L.ptr(t)


def _stream():
    from safepo import _lib as L
    return L.stream()


def _check(key, got, want, scale=None):
    """max |got - want| / scale (default: max |want|) against BAR[key]; entries where want is exactly 0 must be exactly 0."""
    got = torch.as_tensor(got).detach().double().cpu().reshape(-1)
    want = torch.as_tensor(want).detach().double().cpu().reshape(-1)
    assert got.shape == want.shape, (key, got.shape, want.shape)
    assert bool(torch.isfinite(got).all()), key
    zero = want == 0
    assert bool((got[zero] == 0).all()), (key, "nonzero where float64 is exactly 0", got[zero][got[zero] != 0][:8])
    if scale is None:
        scale = float(want.abs().max())
    err = float((got - want).abs().max()) / scale if scale > 0 else float((got - want).abs().max())
    MEASURED[key] = max(MEASURED.get(key, 0.0), err)
    assert err <= BAR[key], (key, err, BAR[key])
    return err


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if MEASURED:
        print("\nmeasured maxima (error / scale) and bars:\n" + "\n".join(f"  {k:12s} {v:.2e}  bar {BAR[k]:.0e}" for k, v in sorted(MEASURED.items())))


# ============================================================ CPU ============================================================
def _branchy_case(g, N=64, D=6, DS=8, A=3, H=16):
    """A small MAPPO-Lag update that reaches every branch: ratios below / inside / above the clip range with both advantage
    signs, the value clip on both sides, all three Huber pieces, the lambda ReLU clamping, weight decay and the norm clip."""
    layer_N = 2
    sts = (_state(g, D, H, A, "actor"), _state(g, DS, H, A, "critic"), _state(g, DS, H, A, "critic"))
    cfg = dict(actor_lr=9e-5, critic_lr=5e-3, opti_eps=1e-5, weight_decay=0.01, clip_param=0.2, huber_delta=0.6, entropy_coef=0.01,
               max_grad_norm=0.05, cost_limit=25.0, gamma=0.96, lagrangian_coef_rate=5.0, value_loss_coef=1.0, lamda_lagr=0.78,
               layer_N=layer_N, std_x_coef=1.0, std_y_coef=0.5)
    s = _sample(g, N, D, DS, A, sts[0], layer_N, 1.0, 0.5, ret_scale=2.0)
    s["old_action_log_probs"] = s["old_action_log_probs"] + 0.5 * torch.randn(N, A, generator=g)     # ratios far outside the range
    s["value_preds"] = 0.8 * torch.randn(N, 1, generator=g)
    s["cost_preds"] = 0.8 * torch.randn(N, 1, generator=g)
    s["aver_episode_costs"] = torch.rand(N, 1, generator=g)       # far below the limit: delta > 0 pushes lambda through 0
    return sts, cfg, s


def test_reference_equals_ma_oracle_bit_for_bit():
    """In float32 the restated MAPPO-Lag update equals OracleMATrainer.ppo_update bit for bit: clipped .grad, weights after
    Adam, the eight returned values, lambda and the PopArt state, on one small case that reaches every branch."""
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        sts, cfg, s = _branchy_case(torch.Generator().manual_seed(11))
        onets = [MA.OracleMANet(st, layer_N=cfg["layer_N"]) for st in sts]
        otr = MA.OracleMATrainer(*onets, cfg)
        want = otr.ppo_update(s)
        got = ref_ppo_update(sts, s, cfg, torch.float32, cfg["layer_N"])
    finally:
        torch.set_num_threads(threads)
    for onet, net in zip(onets, got["nets"]):
        for k, p in onet.p.items():
            assert torch.equal(net[k].grad, p.grad), k
            assert torch.equal(net[k].detach(), p.detach()), k
    for k, v in want.items():
        assert torch.equal(torch.as_tensor(got["out"][k]), torch.as_tensor(v)), k
    assert torch.equal(torch.as_tensor(got["lamda"]), torch.as_tensor(otr.lamda_lagr))
    assert torch.equal(got["popart"].state(), torch.stack([otr.popart.running_mean[0], otr.popart.running_mean_sq[0], otr.popart.debiasing_term]))
    # every branch is present in this case
    imp = got["imp"].reshape(-1)
    adv = (s["adv_targ"] - cfg["lamda_lagr"] * s["cost_adv_targ"]).reshape(-1)
    for region in (imp < 0.8, (imp >= 0.8) & (imp <= 1.2), imp > 1.2):
        for sign in (adv > 0, adv < 0):
            assert int((region & sign).sum()) >= 2
    assert float(got["lamda"]) == 0.0 and cfg["lamda_lagr"] > 0
    for n in (0, 1, 2):
        assert float(torch.cat([g.reshape(-1) for g in got["grads"][n].values()]).norm()) > cfg["max_grad_norm"]
    pa = PopArt(torch.float32)
    d = (s["value_preds"] + 0.0).reshape(-1)
    ret_c = pa.normalize(s["returns"]).reshape(-1)
    ret_o = pa.normalize(s["returns"]).reshape(-1)
    with torch.no_grad():
        v = critic_value(sts[1], s["share_obs"], cfg["layer_N"]).reshape(-1)
    dlt = v - d
    assert int((dlt > 0.2).sum()) >= 2 and int((dlt < -0.2).sum()) >= 2
    for e in (ret_o - v, ret_c - (d + dlt.clamp(-0.2, 0.2))):
        assert int((e > 0.6).sum()) >= 2 and int((e < -0.6).sum()) >= 2 and int((e.abs() <= 0.6).sum()) >= 2


def test_macpo_reference_equals_macpo_oracle_bit_for_bit():
    """In float32 the restated KL, Fisher-vector product, ratio surrogates with their gradients and line-search quantities
    equal tests/macpo_oracle.py's bit for bit."""
    import macpo_oracle as MO
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        g = torch.Generator().manual_seed(12)
        N, D, A, H = 40, 6, 3, 16
        sts = (_state(g, D, H, A, "actor"), _state(g, D, H, A, "critic"), _state(g, D, H, A, "critic"))
        cfg = dict(MA_DEFAULT_CFG(), std_x_coef=X_COEF, std_y_coef=Y_COEF)
        onets = [MA.OracleMANet(st) for st in sts]
        otr = MO.OracleMACPOTrainer(*onets, cfg)
        s = _sample(g, N, D, D, A, sts[0], 2, X_COEF, Y_COEF)
        obs, act = s["obs"], s["actions"]
        v = torch.randn(sum(t.numel() for t in sts[0].values()), generator=g)
        want_fvp = otr.fisher_vector_product(obs, act, v)
        p = {k: t.detach().clone().requires_grad_(True) for k, t in sts[0].items()}
        assert torch.equal(ref_fvp(p, obs, v, 2, X_COEF, Y_COEF), want_fvp)
        lp, _, mu, sd = otr._eval(otr.actor, obs, act)
        rl_o = -torch.sum(torch.prod(torch.exp(lp - s["old_action_log_probs"]), -1, keepdim=True) * s["factor"] * s["adv_targ"], -1, keepdim=True).mean()
        g_o = torch.autograd.grad(rl_o, otr.actor.params())
        dist = actor_dist(p, obs, 2, X_COEF, Y_COEF)
        rl, cl, _ = ratio_surrogates(dist.log_prob(act), s["old_action_log_probs"], s["factor"], s["adv_targ"], s["cost_adv_targ"])
        assert torch.equal(rl, rl_o)
        for a_, b_ in zip(torch.autograd.grad(rl, list(p.values())), g_o):
            assert torch.equal(a_, b_)
        # line search at moved weights against the unmoved actor
        old = MA.OracleMANet(otr.actor.state())
        with torch.no_grad():
            for t in otr.actor.params():
                t.add_(0.01 * torch.randn(t.shape, generator=g))
            kl_o = otr.kl_divergence(obs, act, otr.actor, old).mean()
            new_d = actor_dist(otr.actor.p, obs, 2, X_COEF, Y_COEF)
            old_d = actor_dist(old.p, obs, 2, X_COEF, Y_COEF)
            q = linesearch_quantities(new_d, old_d, act, s["old_action_log_probs"], s["factor"], s["adv_targ"], s["cost_adv_targ"])
            lpn = otr._eval(otr.actor, obs, act)[0]
            ratio = torch.prod(torch.exp(lpn - s["old_action_log_probs"]), dim=-1, keepdim=True)
        assert torch.equal(q[2], kl_o)
        assert torch.equal(q[0], -torch.sum(ratio * s["factor"] * s["adv_targ"], dim=-1, keepdim=True).mean())
        assert torch.equal(q[1], torch.sum(ratio * s["factor"] * s["cost_adv_targ"], dim=-1, keepdim=True).mean())
    finally:
        torch.set_num_threads(threads)


def MA_DEFAULT_CFG():
    from safepo.multi_agent.macpo import DEFAULT_CONFIG
    return dict(DEFAULT_CONFIG)


def test_float64_reference_differentiates_like_float32():
    """The float64 reference of the branchy case stays within float32 rounding of the float32 one (the same branches)."""
    sts, cfg, s = _branchy_case(torch.Generator().manual_seed(11))
    a = ref_ppo_update(sts, s, cfg, torch.float32, cfg["layer_N"])
    b = ref_ppo_update(sts, s, cfg, torch.float64, cfg["layer_N"])
    for ga, gb in zip(a["grads"], b["grads"]):
        for k in ga:
            assert float((ga[k].double() - gb[k]).abs().max()) <= 1e-4 * float(gb[k].abs().max()) + 1e-12, k
    assert b["lamda"].dtype == torch.float64 and float(b["lamda"]) == 0.0


# ============================================================ GPU: per kernel ============================================================
def _layer_inputs(g, n, K, H, lin):
    """Rows with z near 0 (the ELU kink), z << 0, constant and near-constant rows (LayerNorm's eps), and ordinary rows."""
    x = torch.randn(n, K, generator=g)
    kind = torch.arange(n) % 6
    x[kind == 1] *= 1e-4                                  # z ~ b: biases near 0 put z on the kink
    x[kind == 2] *= 30                                    # without the input LayerNorm: |z| large on every column
    x[kind == 3] = 1e-3 * torch.randn(int((kind == 3).sum()), K, generator=g)     # variance ~1e-6 < eps = 1e-5
    x[kind == 4] = 0.5                                    # constant row: exactly zero variance
    if K == 2:
        # LayerNorm over two nearly equal values is ill-conditioned in any fp32 evaluation (x - mean cancels): keep them apart
        close = ((x[:, 0] - x[:, 1]).abs() < 0.1 * x.abs().amax(1)) & (kind != 4)
        x[close, 1] = -x[close, 1]
    W = torch.randn(H, K, generator=g) * (1.4 / K ** 0.5)
    W[H // 8:H // 4] *= 30                                # these columns have |z| >> 1: ELU saturates at -1 on about half the rows
    b = 0.1 * torch.randn(H, generator=g)
    b[:H // 8] = 1e-6 * torch.randn(H // 8, generator=g)
    lw, lb = 1 + 0.1 * torch.randn(H, generator=g), 0.1 * torch.randn(H, generator=g)
    lin_wb = (1 + 0.1 * torch.randn(K, generator=g), 0.1 * torch.randn(K, generator=g)) if lin else None
    return x, W, b, lw, lb, lin_wb


@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 256, 384, 512])
@pytest.mark.parametrize("lin", [False, True])
def test_mlp_layer_vs_float64(H, lin):
    """spo_ma_mlp_layer and spo_ma_mlp_layer_train (out, pre, xn) at K in {2, 18, 66, 398, 512} x n in {1, 31, 33, 4097}."""
    dev = _cuda()
    g = torch.Generator().manual_seed(H + lin)
    for K in (2, 18, 66, 398, 512):
        for n in (1, 31, 33, 4097):
            x, W, b, lw, lb, lwb = _layer_inputs(g, n, K, H, lin)
            d = [t.to(dev).contiguous() for t in (x, W, b, lw, lb)]
            dl = [t.to(dev).contiguous() for t in lwb] if lin else [None, None]
            out, out2, pre = (torch.empty(n, H, device=dev) for _ in range(3))
            xn = torch.empty(n, K, device=dev) if lin else None
            _call("spo_ma_mlp_layer", _ptr(d[0]), n, K, _ptr(d[1]), _ptr(d[2]), _ptr(d[3]), _ptr(d[4]), H, _ptr(dl[0]), _ptr(dl[1]), _ptr(out), _stream())
            _call("spo_ma_mlp_layer_train", _ptr(d[0]), n, K, _ptr(d[1]), _ptr(d[2]), _ptr(d[3]), _ptr(d[4]), H, _ptr(dl[0]), _ptr(dl[1]),
                  _ptr(out2), _ptr(pre), _ptr(xn), _stream())
            torch.cuda.synchronize()
            x64 = x.double()
            xin = ln(x64, *[t.double() for t in lwb]) if lin else x64
            z = F.linear(xin, W.double(), b.double())
            pre64 = F.elu(z)
            want = ln(pre64, lw.double(), lb.double())
            _check("layer", out, want)
            assert torch.equal(out, out2), (H, K, n)
            _check("layer", pre, pre64)
            if lin:
                _check("layer", xn, xin)
            if n == 4097:
                assert int((z.abs() < 1e-3).sum()) >= H // 8 and int((z < -10).sum()) >= n * H // 64, (H, K, n)


@pytest.mark.gpu
def test_mlp_layer_rejects_odd_k_as_unsupported():
    """Odd obs_dim and H off the 128 grid are refused with SPO_ERR_UNSUPPORTED before any launch."""
    from safepo import _lib as L
    dev = _cuda()
    x, W = torch.zeros(4, 8, device=dev), torch.zeros(640, 8, device=dev)
    v, out = torch.zeros(640, device=dev), torch.zeros(4, 640, device=dev)
    for K, H in ((7, 128), (8, 640), (8, 192)):
        rc = L.lib().spo_ma_mlp_layer(_ptr(x), 4, K, _ptr(W), _ptr(v), _ptr(v), _ptr(v), H, None, None, _ptr(out), _stream())
        assert rc == -2, (K, H, rc)


@pytest.mark.gpu
@pytest.mark.parametrize("A", [1, 20, 32])
def test_head_vs_float64(A):
    """spo_ma_head: the DiagGaussian head sampled and deterministic with per-dimension log-probs (std_x_coef != 1), and the
    value head."""
    dev = _cuda()
    g = torch.Generator().manual_seed(100 + A)
    for n, H in ((1, 128), (33, 384), (1000, 512)):
        feat = torch.randn(n, H, generator=g)
        W, b = torch.randn(A, H, generator=g) * 0.05, 0.1 * torch.randn(A, generator=g)
        ls, eps = torch.randn(A, generator=g), torch.randn(n, A, generator=g)
        fd, Wd, bd, lsd, ed = (t.to(dev).contiguous() for t in (feat, W, b, ls, eps))
        mean64 = F.linear(feat.double(), W.double(), b.double())
        dist = diag_gaussian(mean64, ls.double(), X_COEF, Y_COEF)
        for sampled in (True, False):
            out, logp = torch.empty(n, A, device=dev), torch.empty(n, A, device=dev)
            _call("spo_ma_head", _ptr(fd), n, H, _ptr(Wd), _ptr(bd), A, _ptr(lsd), X_COEF, Y_COEF, _ptr(ed) if sampled else None, _ptr(out),
                  _ptr(logp), _stream())
            torch.cuda.synchronize()
            act64 = mean64 + dist.stddev * eps.double() if sampled else mean64
            _check("head", out, act64)
            _check("head", logp, dist.log_prob(act64))
        v, W1 = torch.empty(n, 1, device=dev), Wd[:1].clone()
        _call("spo_ma_head", _ptr(fd), n, H, _ptr(W1), _ptr(bd), 1, None, 1.0, 1.0, None, _ptr(v), None, _stream())
        torch.cuda.synchronize()
        _check("head", v, F.linear(feat.double(), W[:1].double(), b[:1].double()))


def _reduce(part, nblk, stride, nseg, length, outs, scale=1.0):
    _call("spo_ma_partial_reduce", _ptr(part), nblk, stride, nseg, length, *[_ptr(o) for o in outs], scale, _stream())


@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 256, 384, 512])
def test_ln_elu_bwd_and_partial_reduce_vs_float64(H):
    """spo_ma_ln_elu_bwd: dz and the three column sums (d gamma, d beta, d bias) through spo_ma_partial_reduce with nseg 1-3
    and null outputs left untouched, n in {1, 31, 33, 1000}."""
    dev = _cuda()
    g = torch.Generator().manual_seed(200 + H)
    for n in (1, 31, 33, 1000):
        z = torch.randn(n, H, generator=g) * 2
        z[:, :4] = 0.0                                   # on the kink: ELU'(0) = 1 on both sides
        pre = F.elu(z)
        dy, lw = torch.randn(n, H, generator=g), 1 + 0.2 * torch.randn(H, generator=g)
        lb = 0.1 * torch.randn(H, generator=g)
        dyd, pred, lwd = (t.to(dev).contiguous() for t in (dy, pre, lw))
        nb = (n + 31) // 32
        dz, part = torch.empty(n, H, device=dev), torch.empty(nb * 3 * H, device=dev)
        _call("spo_ma_ln_elu_bwd", _ptr(dyd), _ptr(pred), _ptr(lwd), n, H, _ptr(dz), _ptr(part), _stream())
        # float64: z from pre (ELU is invertible), autograd of LN(ELU(z)) * gamma + beta against dy
        z64 = torch.where(pre.double() > 0, pre.double(), torch.log1p(pre.double())).requires_grad_(True)
        lw64, lb64 = lw.double().requires_grad_(True), lb.double().requires_grad_(True)
        y = ln(F.elu(z64), lw64, lb64)
        dz64, dg64, db64 = torch.autograd.grad((y * dy.double()).sum(), (z64, lw64, lb64))
        outs = [torch.full((H,), 7.0, device=dev) for _ in range(3)]
        _reduce(part, nb, 3 * H, 3, H, outs)
        torch.cuda.synchronize()
        _check("ln_bwd", dz, dz64)
        for o, w in zip(outs, (dg64, db64, dz64.sum(0))):
            _check("ln_bwd", o, w)
        for nseg, null in ((3, 1), (2, 0), (1, None)):
            o2 = [torch.full((H,), 7.0, device=dev) for _ in range(3)]
            ptrs = [o2[i] if i < nseg and i != null else None for i in range(3)]
            _reduce(part, nb, 3 * H, nseg, H, ptrs, scale=0.5)
            torch.cuda.synchronize()
            for i in range(3):
                if ptrs[i] is None:
                    assert bool((o2[i] == 7.0).all()), (nseg, null, i)
                else:
                    assert torch.equal(o2[i], outs[i] * 0.5), (nseg, i)


@pytest.mark.gpu
@pytest.mark.parametrize("K", [2, 66, 398])
def test_ln_in_bwd_vs_float64(K):
    """spo_ma_ln_in_bwd: the input LayerNorm's weight / bias gradients, with near-constant rows where its eps matters."""
    dev = _cuda()
    g = torch.Generator().manual_seed(300 + K)
    for n in (1, 31, 33, 1000):
        x = torch.randn(n, K, generator=g) * 2 + 0.5
        x[1::3] = 1e-3 * torch.randn(len(range(1, n, 3)), K, generator=g)      # variance ~1e-6 < eps = 1e-5
        dxn = torch.randn(n, K, generator=g)
        w, b = (1 + 0.1 * torch.randn(K, generator=g)).double().requires_grad_(True), (0.1 * torch.randn(K, generator=g)).double().requires_grad_(True)
        gw, gb = torch.autograd.grad((ln(x.double(), w, b) * dxn.double()).sum(), (w, b))
        xd, dd = x.to(dev), dxn.to(dev)
        nb = (n + 31) // 32
        part = torch.empty(nb * 2 * K, device=dev)
        _call("spo_ma_ln_in_bwd", _ptr(dd), _ptr(xd), n, K, _ptr(part), _stream())
        outs = [torch.empty(K, device=dev) for _ in range(2)]
        _reduce(part, nb, 2 * K, 2, K, outs + [None])
        torch.cuda.synchronize()
        _check("ln_bwd", outs[0], gw)
        _check("ln_bwd", outs[1], gb)


def _actor_loss_case(g, n, A, H, lam, clip):
    """Inputs whose importance weights fall below / inside / above the clip range (margin >= 0.05) for both signs of the
    mixed advantage, and rows whose mixed advantage is exactly 0."""
    feat = torch.randn(n, H, generator=g)
    W, b = torch.randn(A, H, generator=g) * 0.05, 0.1 * torch.randn(A, generator=g)
    ls = 0.5 * torch.randn(A, generator=g)
    with torch.no_grad():
        dist = diag_gaussian(F.linear(feat.double(), W.double(), b.double()), ls.double(), X_COEF, Y_COEF)
        actions = (dist.mean + dist.stddev * torch.randn(n, A, generator=g, dtype=torch.float64)).float()
        lp64 = dist.log_prob(actions.double())
    r = torch.arange(n)
    region, sign = r % 3, torch.where((r // 3) % 2 == 0, 1.0, -1.0)
    lo, hi = 1 - clip, 1 + clip
    u = torch.rand(n, generator=g, dtype=torch.float64)
    target = torch.where(region == 0, lo - 0.25 + 0.2 * u, torch.where(region == 1, lo + 0.05 + (hi - lo - 0.1) * u, hi + 0.05 + 0.3 * u))
    old = (lp64 - torch.log(target)[:, None] / A).float()
    cadv = torch.randn(n, generator=g)
    hyb = sign * (0.3 + torch.rand(n, generator=g))
    adv = (hyb + lam * cadv)
    zero = r % 7 == 5
    adv[zero] = lam * cadv[zero]                       # exact in fp32 and float64 (lam = 0.5): adv - lam * cadv == 0
    factor = torch.rand(n, generator=g) + 0.5
    return feat, W, b, ls, actions, old, adv, cadv, factor, region, zero


@pytest.mark.gpu
@pytest.mark.parametrize("A", [1, 2, 20, 31, 32])
def test_actor_loss_vs_float64(A):
    """spo_ma_actor_loss + spo_ma_actor_finalize: dmean per element, the importance weights, g_b, g_log_std (with the entropy
    bonus), the policy loss and the entropy at n in {1, 33, 1000}, lambda > 0; every clip case populated."""
    dev = _cuda()
    g = torch.Generator().manual_seed(400 + A)
    lam, clip, ec, H = 0.5, 0.2, 0.013, 384
    for n in (1, 33, 1000):
        feat, W, b, ls, actions, old, adv, cadv, factor, region, zero = _actor_loss_case(g, n, A, H, lam, clip)
        args = [t.to(dev).contiguous() for t in (feat, W, b, ls, actions, old, adv, cadv, factor)]
        lamd = torch.tensor([lam], device=dev)
        nb = (n + 31) // 32
        dmean, imp, part = torch.empty(n, A, device=dev), torch.empty(n, device=dev), torch.empty(nb * 66, device=dev)
        _call("spo_ma_actor_loss", _ptr(args[0]), n, H, _ptr(args[1]), _ptr(args[2]), _ptr(args[3]), A, _ptr(args[4]), _ptr(args[5]),
              _ptr(args[6]), _ptr(args[7]), _ptr(args[8]), _ptr(lamd), 1.0 - clip, 1.0 + clip, X_COEF, Y_COEF, _ptr(dmean), _ptr(imp),
              _ptr(part), _stream())
        gb, gls, scal = torch.empty(A, device=dev), torch.empty(A, device=dev), torch.empty(2, device=dev)
        _call("spo_ma_actor_finalize", _ptr(part), nb, n, _ptr(args[3]), A, X_COEF, Y_COEF, ec, _ptr(gb), _ptr(gls), _ptr(scal), _stream())
        torch.cuda.synchronize()
        mean = F.linear(feat.double(), W.double(), b.double()).requires_grad_(True)
        ls64 = ls.double().requires_grad_(True)
        dist = diag_gaussian(mean, ls64, X_COEF, Y_COEF)
        pl, imp64 = surrogate(dist.log_prob(actions.double()), old.double(), adv.double()[:, None], cadv.double()[:, None],
                              factor.double()[:, None], lam, clip)
        ent = dist.entropy().mean()
        (dm64,) = torch.autograd.grad(pl, mean, retain_graph=True)
        (gls64,) = torch.autograd.grad(pl - ent * ec, ls64)
        imp64 = imp64.detach().reshape(-1)
        # the same branch on both sides, and every branch populated
        cat = lambda t: (t < 1 - clip).int() + 2 * (t > 1 + clip).int()      # noqa: E731
        assert torch.equal(cat(imp.cpu().double()), cat(imp64)) and torch.equal(cat(imp64), torch.tensor([1, 0, 2], dtype=torch.int32)[region])
        if n >= 33:
            hyb = adv.double() - lam * cadv.double()
            for reg in (0, 1, 2):
                for sgn in (hyb > 0, hyb < 0):
                    assert int(((region == reg) & sgn).sum()) >= n // 10, (reg, n)
            assert int(zero.sum()) >= 4 and bool((hyb[zero] == 0).all())
        _check("actor", dmean, dm64)
        _check("actor", imp, imp64)
        _check("actor", gb, dm64.sum(0))
        _check("actor", gls, gls64)
        terms = factor.double() * torch.minimum(imp64 * hyb_of(adv, cadv, lam), imp64.clamp(1 - clip, 1 + clip) * hyb_of(adv, cadv, lam))
        _check("actor_loss", scal[0:1], pl.detach().reshape(1), scale=float(terms.abs().mean()) + 1e-30)
        _check("actor_loss", scal[1:2], ent.detach().reshape(1))


def hyb_of(adv, cadv, lam):
    return adv.double() - lam * cadv.double()


def _value_case(n_rows=None):
    """Exactly representable rows (multiples of 1/8): value difference below / at / inside / at / above +-clip (clip 0.25),
    errors in all three Huber pieces (delta 2, including +-delta itself), and ties huber(eo) == huber(ec)."""
    dlts = [-0.75, -0.25, -0.125, 0.0, 0.125, 0.25, 0.75]
    errs = [-3.0, -2.5, -2.0, -1.5, -0.5, 0.0, 0.5, 1.5, 2.0, 2.5, 3.0]
    rows = [(d, ec, eo) for d in dlts for ec in errs for eo in errs]
    g = torch.Generator().manual_seed(17)
    perm = torch.randperm(len(rows), generator=g)
    rows = [rows[i] for i in perm[:n_rows]] if n_rows else [rows[i] for i in perm]
    n = len(rows)
    dlt, ec, eo = (torch.tensor([r[i] for r in rows], dtype=torch.float64) for i in range(3))
    vp = torch.randint(-8, 9, (n,), generator=g).double() / 8
    v = vp + dlt
    rn_c, rn_o = vp + dlt.clamp(-0.25, 0.25) + ec, v + eo
    return v, vp, rn_c, rn_o, dlt, ec, eo


@pytest.mark.gpu
def test_value_loss_every_branch_vs_float64():
    """spo_ma_value_loss: every Huber piece on both errors, the value clip on both sides and exactly at +-clip, torch.max ties."""
    dev = _cuda()
    clip, d = 0.25, 2.0
    for n_rows in (1, 300, None):
        v, vp, rn_c, rn_o, dlt, ec, eo = _value_case(n_rows)
        n = v.numel()
        ins = [t.float().to(dev) for t in (v, vp, rn_c, rn_o)]
        assert all(torch.equal(a.cpu().double(), b) for a, b in zip(ins, (v, vp, rn_c, rn_o)))     # exactly representable
        nb = (n + 255) // 256
        dv, part, loss, sdv = torch.empty(n, device=dev), torch.empty(nb * 2, device=dev), torch.empty(1, device=dev), torch.empty(1, device=dev)
        coef = 1.0
        _call("spo_ma_value_loss", *[_ptr(t) for t in ins], n, clip, d, coef / n, _ptr(dv), _ptr(part), _stream())
        _reduce(part, nb, 2, 1, 1, [loss, None, None], 1.0 / n)
        _reduce(part, nb, 2, 2, 1, [None, sdv, None])
        torch.cuda.synchronize()
        v64 = v.clone().requires_grad_(True)
        L = value_loss(v64, vp, rn_c, rn_o, clip, d)
        (dv64,) = torch.autograd.grad(L * coef, v64)
        _check("value", dv, dv64)
        _check("value", sdv, dv64.sum().reshape(1), scale=float(dv64.abs().sum()))
        _check("value", loss, L.detach().reshape(1))
        if n_rows is None:
            ho, hc = huber(eo, d), huber(ec, d)
            counts = dict(ec_quad=(ec.abs() <= d), ec_lin=(ec > d), ec_zero=(ec < -d), eo_quad=(eo.abs() <= d), eo_lin=(eo > d), eo_zero=(eo < -d),
                          clip_hi=(dlt > clip), clip_lo=(dlt < -clip), at_hi=(dlt == clip), at_lo=(dlt == -clip), inside=(dlt.abs() < clip),
                          tie=(ho == hc), tie_nonzero=(ho == hc) & (ho > 0), ho_wins=(ho > hc), hc_wins=(ho < hc))
            for k, m in counts.items():
                assert int(m.sum()) >= 40, (k, int(m.sum()))
            # the tie rows' gradient is half of each side's (torch.max's rule): a nonzero share of them
            assert int(((ho == hc) & (dv64 != 0)).sum()) >= 20


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 1023, 1025, 100000])
def test_popart_vs_float64(n):
    """spo_ma_popart_normalize, two calls in a row (the reference normalises twice per value loss): state and outputs."""
    dev = _cuda()
    g = torch.Generator().manual_seed(500 + n)
    st = torch.zeros(3, device=dev)
    pa = PopArt(torch.float64)
    for call in range(2):
        x = torch.randn(n, generator=g) * 3 + 1 + call
        xd, out = x.to(dev), torch.empty(n, device=dev)
        _call("spo_ma_popart_normalize", _ptr(xd), n, _ptr(st), 0.99999, 1e-5, _ptr(out), _stream())
        torch.cuda.synchronize()
        want = pa.normalize(x.double()[:, None]).reshape(-1)
        _check("popart", st, pa.state())
        sd = float(torch.sqrt((pa.running_mean_sq / pa.debiasing_term - (pa.running_mean / pa.debiasing_term) ** 2).clamp(min=1e-2)))
        _check("popart", out, want, scale=float(x.abs().max()) / sd)


@pytest.mark.gpu
@pytest.mark.parametrize("clamps", [False, True])
def test_lagrange_step_vs_float64(clamps):
    """spo_ma_lagrange_step: lambda <- relu(lambda - delta rate), with the ReLU clamping and not."""
    dev = _cuda()
    g = torch.Generator().manual_seed(600 + clamps)
    for n in (1, 1000, 5000):
        imp, cadv = torch.rand(n, generator=g) + 0.5, 0.1 * torch.randn(n, generator=g)
        aver = torch.rand(n, generator=g) * 10 if clamps else torch.rand(n, generator=g) * 10 + 60
        lam0, rate, limit, gamma = 0.3, 2.0, 25.0, 0.96
        lamd = torch.tensor([lam0], device=dev)
        ins = [t.to(dev) for t in (imp, cadv, aver)]
        _call("spo_ma_lagrange_step", *[_ptr(t) for t in ins], n, limit, gamma, rate, _ptr(lamd), _stream())
        torch.cuda.synchronize()
        want = lagrange_step(lam0, imp.double(), cadv.double(), aver.double(), limit, gamma, rate)
        unclamped = lam0 - float(-((aver.double().mean() - limit) * (1 - gamma) + imp.double() * cadv.double()).mean()) * rate
        assert (unclamped < -0.1) if clamps else (unclamped > 0.1), unclamped
        if clamps:
            assert float(lamd) == 0.0 and float(want) == 0.0
        _check("lagrange", lamd, want.reshape(1), scale=abs(unclamped) + lam0)


@pytest.mark.gpu
@pytest.mark.parametrize("count", [1, 257, 1024 * 256 + 4099])
def test_clip_adam_vs_float64(count):
    """spo_ma_clip_adam: the grid-stride sum of squares, the clip active and not, weight decay != 0, steps 1 and 7, against
    clip_grad_norm_ + torch.optim.Adam on float64 copies."""
    dev = _cuda()
    g = torch.Generator().manual_seed(700 + count)
    lr, eps, wd = 1e-3, 1e-5, 0.5
    for step in (1, 7):
        for active in (False, True):
            p = 0.01 * torch.randn(count, generator=g)
            # |g| >= 0.5 keeps the decayed, clipped gradient far from 0, where Adam's g / (|g| + eps) is ill-conditioned in fp32
            grad = torch.where(torch.rand(count, generator=g) < 0.5, -1.0, 1.0) * (0.5 + torch.rand(count, generator=g))
            norm64 = float(grad.double().norm())
            max_norm = 0.3 * norm64 if active else 3.0 * norm64
            m0 = torch.zeros(count) if step == 1 else 0.1 * torch.randn(count, generator=g)
            v0 = torch.zeros(count) if step == 1 else m0 ** 2 + 0.01 * torch.rand(count, generator=g)
            pd, gd, md, vd = (t.to(dev).contiguous() for t in (p, grad, m0, v0))
            work, norm = torch.empty(1024, device=dev), torch.empty(2, device=dev)
            _call("spo_ma_clip_adam", _ptr(pd), _ptr(gd), _ptr(md), _ptr(vd), count, max_norm, lr, 0.9, 0.999, eps, wd, step, _ptr(work), _ptr(norm),
                  _stream())
            torch.cuda.synchronize()
            p64 = p.double().clone().requires_grad_(True)
            p64.grad = grad.double().clone()
            state = None if step == 1 else [(step - 1, m0.double(), v0.double())]
            opt_norm, opt = clip_adam([p64], lr, eps, wd, max_norm, state)
            coef = min(1.0, max_norm / (norm64 + 1e-6))
            assert (coef < 0.5) if active else coef == 1.0
            _check("adam", norm[0:1], opt_norm.reshape(1))
            _check("adam", norm[1:2], torch.tensor([coef], dtype=torch.float64))
            # the weights relative to their movement (p is O(1e-2), so fp32 rounding of p is far below lr)
            _check("adam", pd.cpu().double() - p.double(), p64.detach() - p.double())
            _check("adam", md, opt.state[p64]["exp_avg"])
            _check("adam", vd, opt.state[p64]["exp_avg_sq"])


def _valid_slices(R, want):
    s = want
    while s > 1 and (s - 1) * (((R + s - 1) // s + 31) // 32 * 32) >= R:
        s -= 1
    return s


@pytest.mark.gpu
@pytest.mark.parametrize("R,M,N,slices", [(1000, 1, 384, 32), (1000, 20, 1, 32), (4097, 128, 65, 17), (4097, 1, 1, 32), (993, 384, 33, 32),
                                          (31, 7, 5, 1)])
def test_gemm_tn_slices_vs_float64(R, M, N, slices):
    """spo_ma_gemm_tn + spo_ma_partial_reduce: up to 32 row slices with R not a multiple of 32, M or N = 1."""
    dev = _cuda()
    g = torch.Generator().manual_seed(R + M + N)
    A_, B_ = torch.randn(R, M, generator=g), torch.randn(R, N, generator=g)
    Ad, Bd = A_.to(dev), B_.to(dev)
    s = _valid_slices(R, slices)
    assert s == slices or R == 4097, (R, s)
    part, out = torch.empty(s * M * N, device=dev), torch.empty(M, N, device=dev)
    _call("spo_ma_gemm_tn", _ptr(Ad), _ptr(Bd), _ptr(part), R, M, N, s, _stream())
    _reduce(part, s, M * N, 1, M * N, [out, None, None])
    torch.cuda.synchronize()
    _check("gemm", out, A_.double().t() @ B_.double())


@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 384])
@pytest.mark.parametrize("lin", [False, True])
def test_mlp_layer_jvp_vs_float64(H, lin):
    """spo_ma_mlp_layer_jvp against float64 torch.func.jvp of the block, K in {2, 66}, n in {1, 33}."""
    dev = _cuda()
    g = torch.Generator().manual_seed(800 + H + lin)
    for K in (2, 66):
        for n in (1, 33):
            x, W, b, lw, lb, lwb = _layer_inputs(g, n, K, H, lin)
            din = torch.randn(n, K, generator=g)
            dW, db, dlw, dlb = 0.1 * torch.randn(H, K, generator=g), 0.1 * torch.randn(H, generator=g), 0.1 * torch.randn(H, generator=g), 0.1 * torch.randn(H, generator=g)
            dlin = (0.1 * torch.randn(K, generator=g), 0.1 * torch.randn(K, generator=g)) if lin else None
            d = {k: t.to(dev).contiguous() for k, t in dict(x=x, W=W, b=b, lw=lw, lb=lb, din=din, dW=dW, db=db, dlw=dlw, dlb=dlb).items()}
            dl = [t.to(dev).contiguous() for t in (lwb + dlin)] if lin else [None] * 4
            out, pre, dout = (torch.empty(n, H, device=dev) for _ in range(3))
            _call("spo_ma_mlp_layer_train", _ptr(d["x"]), n, K, _ptr(d["W"]), _ptr(d["b"]), _ptr(d["lw"]), _ptr(d["lb"]), H, _ptr(dl[0]), _ptr(dl[1]),
                  _ptr(out), _ptr(pre), None, _stream())
            _call("spo_ma_mlp_layer_jvp", _ptr(d["x"]), None if lin else _ptr(d["din"]), n, K, _ptr(d["W"]), _ptr(d["dW"]), _ptr(d["db"]), _ptr(pre),
                  _ptr(d["lw"]), _ptr(d["dlw"]), _ptr(d["dlb"]), H, *[_ptr(t) for t in dl], _ptr(dout), _stream())
            torch.cuda.synchronize()
            prim = [t.double() for t in (x, W, b, lw, lb)] + ([t.double() for t in lwb] if lin else [])
            tang = [torch.zeros(n, K, dtype=torch.float64) if lin else din.double()] + [t.double() for t in (dW, db, dlw, dlb)] + \
                ([t.double() for t in dlin] if lin else [])

            def fn(xx, W_, b_, lw_, lb_, *li):
                return block(xx, W_, b_, lw_, lb_, tuple(li) if li else None)
            _, want = torch.func.jvp(fn, tuple(prim), tuple(tang))
            _check("jvp", dout, want)


@pytest.mark.gpu
@pytest.mark.parametrize("A", [1, 32])
def test_head_jvp_vs_float64(A):
    """spo_ma_head_jvp: the mean tangent times the Hessian of the reference's mean KL along the means (float64 double
    backprop), and its column sums, H in {128, 384}, n in {1, 33}."""
    dev = _cuda()
    g = torch.Generator().manual_seed(900 + A)
    for H in (128, 384):
        for n in (1, 33):
            feat, dfeat = torch.randn(n, H, generator=g), torch.randn(n, H, generator=g)
            W, dW = torch.randn(A, H, generator=g) * 0.05, 0.1 * torch.randn(A, H, generator=g)
            b, db, ls = 0.1 * torch.randn(A, generator=g), 0.1 * torch.randn(A, generator=g), torch.randn(A, generator=g)
            d = [t.to(dev).contiguous() for t in (feat, dfeat, W, dW, db, ls)]
            nb = (n + 31) // 32
            dmean, part, colsum = torch.empty(n, A, device=dev), torch.empty(nb * A, device=dev), torch.empty(A, device=dev)
            _call("spo_ma_head_jvp", _ptr(d[0]), _ptr(d[1]), n, H, _ptr(d[2]), _ptr(d[3]), _ptr(d[4]), A, _ptr(d[5]), X_COEF, Y_COEF, _ptr(dmean),
                  _ptr(part), _stream())
            _reduce(part, nb, A, 1, A, [colsum, None, None])
            torch.cuda.synchronize()
            _, t = torch.func.jvp(lambda f, w_, b_: F.linear(f, w_, b_), (feat.double(), W.double(), b.double()), (dfeat.double(), dW.double(), db.double()))
            mu0 = F.linear(feat.double(), W.double(), b.double())
            std = torch.sigmoid(ls.double() / X_COEF) * Y_COEF
            mu = mu0.clone().requires_grad_(True)
            kl = kl_terms(mu, std.expand(n, A), mu0, std.expand(n, A)).mean()
            (gk,) = torch.autograd.grad(kl, mu, create_graph=True)
            (want,) = torch.autograd.grad((gk * t).sum(), mu)
            _check("head_jvp", dmean, want)
            _check("head_jvp", colsum, want.sum(0))


def _ratio_inputs(g, n, A):
    mean, ls = torch.randn(n, A, generator=g), 0.5 * torch.randn(A, generator=g)
    std = torch.sigmoid(ls.double() / X_COEF) * Y_COEF
    actions = (mean.double() + std * torch.randn(n, A, generator=g, dtype=torch.float64)).float()
    old = (Normal(mean.double(), std).log_prob(actions.double()) + 0.1 * torch.randn(n, A, generator=g, dtype=torch.float64) / A ** 0.5).float()
    adv, cadv, factor = torch.randn(n, generator=g), torch.randn(n, generator=g), torch.rand(n, generator=g) + 0.5
    return mean, ls, actions, old, adv, cadv, factor


@pytest.mark.gpu
@pytest.mark.parametrize("A", [1, 32])
def test_ratio_loss_and_linesearch_eval_vs_float64(A):
    """spo_ma_ratio_loss (loss, dmean, g_b, g_log_std for both signs) and spo_ma_linesearch_eval (reward / cost loss, KL, mean
    ratio), n in {1, 31, 32, 33, 1000}."""
    dev = _cuda()
    g = torch.Generator().manual_seed(1000 + A)
    for n in (1, 31, 32, 33, 1000):
        mean, ls, actions, old, adv, cadv, factor = _ratio_inputs(g, n, A)
        d = [t.to(dev).contiguous() for t in (mean, ls, actions, old, adv, cadv, factor)]
        nb = (n + 31) // 32
        for sign, a_d, a_ in ((-1.0, d[4], adv), (1.0, d[5], cadv)):
            dmean, part = torch.empty(n, A, device=dev), torch.empty(nb * 3 * A, device=dev)
            loss, gb, gls = torch.empty(A, device=dev), torch.empty(A, device=dev), torch.empty(A, device=dev)
            _call("spo_ma_ratio_loss", _ptr(d[0]), n, _ptr(d[1]), A, _ptr(d[2]), _ptr(d[3]), _ptr(a_d), _ptr(d[6]), sign, X_COEF, Y_COEF, _ptr(dmean),
                  _ptr(part), _stream())
            _reduce(part, nb, 3 * A, 1, A, [loss, None, None], sign / n)
            _reduce(part, nb, 3 * A, 3, A, [None, gb, gls])
            torch.cuda.synchronize()
            mu, ls64 = mean.double().requires_grad_(True), ls.double().requires_grad_(True)
            lp = diag_gaussian(mu, ls64, X_COEF, Y_COEF).log_prob(actions.double())
            rl, cl, ratio = ratio_surrogates(lp, old.double(), factor.double()[:, None], a_.double()[:, None], a_.double()[:, None])
            L = rl if sign < 0 else cl
            dm64, gls64 = torch.autograd.grad(L, (mu, ls64))
            term_scale = float((ratio.detach().reshape(-1) * factor.double() * a_.double()).abs().mean())
            _check("ratio", loss[0:1], L.detach().reshape(1), scale=term_scale)
            _check("ratio", dmean, dm64)
            _check("ratio", gb, dm64.sum(0))
            _check("ratio", gls, gls64)
        # line search: new means / log_std moved from the old ones
        mean_new, ls_new = mean + 0.05 * torch.randn(n, A, generator=g), ls + 0.05 * torch.randn(A, generator=g)
        dn = [t.to(dev).contiguous() for t in (mean_new, ls_new)]
        work, out = torch.zeros(_work_floats(), device=dev), torch.empty(4, device=dev)
        _call("spo_ma_linesearch_eval", _ptr(dn[0]), _ptr(d[0]), _ptr(dn[1]), _ptr(d[1]), A, _ptr(d[2]), _ptr(d[3]), _ptr(d[4]), _ptr(d[5]), _ptr(d[6]),
              n, X_COEF, Y_COEF, _ptr(work), _ptr(out), _stream())
        torch.cuda.synchronize()
        new = diag_gaussian(mean_new.double(), ls_new.double(), X_COEF, Y_COEF)
        oldd = diag_gaussian(mean.double(), ls.double(), X_COEF, Y_COEF)
        q = linesearch_quantities(new, oldd, actions.double(), old.double(), factor.double()[:, None], adv.double()[:, None], cadv.double()[:, None])
        ratio = torch.prod(torch.exp(new.log_prob(actions.double()) - old.double()), -1)
        for i, a_ in ((0, adv), (1, cadv)):
            _check("ls_loss", out[i:i + 1], q[i].reshape(1), scale=float((ratio * factor.double() * a_.double()).abs().mean()))
        _check("ls_loss", out[3:4], q[3].reshape(1))
        # the KL is a sum of A terms of size ~1/2 that cancel: relative to the size of those terms
        kl_scale = float((new.stddev.log() - oldd.stddev.log()).abs().sum(1).mean() + A * 0.5 * 2)
        _check("ls_kl", out[2:3], q[2].reshape(1), scale=kl_scale)


def _work_floats():
    from safepo import _lib as L
    return L.lib().spo_ma_work_floats()


@pytest.mark.gpu
@pytest.mark.parametrize("A", [1, 32])
@pytest.mark.parametrize("at_end", [False, True])
def test_fvp_finalize_vs_float64(A, at_end):
    """spo_ma_fvp_finalize: the log_std block from float64 double backprop of the reference's KL, damping elsewhere, the
    block at offset 0 and at P - A, zero padding kept exactly 0."""
    dev = _cuda()
    g = torch.Generator().manual_seed(1100 + A + at_end)
    P = 1000 + A
    gn, v = torch.randn(P, generator=g), torch.randn(P, generator=g)
    off = P - A if at_end else 0
    pad = torch.zeros(P, dtype=torch.bool)
    pad[(off + A + 3) % P:(off + A + 3) % P + 3] = True
    gn[pad], v[pad] = 0.0, 0.0
    ls = 1.5 * torch.randn(A, generator=g)
    d = [t.to(dev).contiguous() for t in (gn, v, ls)]
    out = torch.empty(P, device=dev)
    _call("spo_ma_fvp_finalize", _ptr(d[0]), _ptr(d[1]), _ptr(out), P, _ptr(d[2]), off, A, X_COEF, Y_COEF, 0.1, _stream())
    torch.cuda.synchronize()
    l64 = ls.double().requires_grad_(True)
    std = torch.sigmoid(l64 / X_COEF) * Y_COEF
    mu = torch.zeros(1, A, dtype=torch.float64)
    kl = kl_terms(mu, std[None], mu, std[None].detach()).mean()
    (gk,) = torch.autograd.grad(kl, l64, create_graph=True)
    (hv,) = torch.autograd.grad((gk * v[off:off + A].double()).sum(), l64)
    want = gn.double() + 0.1 * v.double()
    want[off:off + A] = hv + 0.1 * v[off:off + A].double()
    _check("finalize", out, want)
    _check("finalize", out[off:off + A], want[off:off + A])
    assert bool((out.cpu()[pad] == 0).all())


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 255, 256 * 256 + 1])
def test_vector_kernels_vs_float64(P):
    """spo_ma_dots (1-4 pairs), spo_ma_cg_begin / _update (a step, the stop flag, a stopped solve left bit-identical),
    spo_ma_step_dir (both modes), spo_ma_ls_trial (|x| above and below 0.5); padding stays exactly 0."""
    dev = _cuda()
    g = torch.Generator().manual_seed(1200 + P)
    pad = torch.zeros(P, dtype=torch.bool)
    if P > 8:
        pad[P // 3:P // 3 + 5] = True

    def vec(scale=1.0):
        t = torch.randn(P, generator=g) * scale
        t[pad] = 0.0
        return t
    work = torch.zeros(_work_floats(), device=dev)
    # ---- dots ----
    for ndot in (1, 2, 3, 4):
        a = [vec() for _ in range(ndot)]
        b = [vec() for _ in range(ndot)]
        ad, bd = [t.to(dev) for t in a], [t.to(dev) for t in b]
        ptrs = []
        for i in range(4):
            ptrs += [_ptr(ad[i]), _ptr(bd[i])] if i < ndot else [None, None]
        out = torch.empty(4, device=dev)
        _call("spo_ma_dots", *ptrs, ndot, P, _ptr(work), _ptr(out), _stream())
        torch.cuda.synchronize()
        for i in range(ndot):
            prod = a[i].double() * b[i].double()
            _check("vec", out[i:i + 1], prod.sum().reshape(1), scale=float(prod.abs().sum()))
    # ---- CG: begin, one step, then a step that sets the stop flag, then a stopped step; Ap = D p with D > 0 diagonal ----
    bvec, dg = vec(), 0.5 + torch.rand(P, generator=g)
    bd, dgd = bvec.to(dev), dg.to(dev)
    Apd = torch.empty(P, device=dev)
    x, r, p = torch.full((P,), 3.0, device=dev), torch.empty(P, device=dev), torch.empty(P, device=dev)
    st = torch.full((4,), 5.0, device=dev)
    _call("spo_ma_cg_begin", _ptr(bd), _ptr(x), _ptr(r), _ptr(p), P, _ptr(work), _ptr(st), _stream())
    torch.cuda.synchronize()
    assert bool((x == 0).all()) and torch.equal(r, bd) and torch.equal(p, bd)
    _check("vec", st[0:1], (bvec.double() ** 2).sum().reshape(1))
    assert torch.equal(st[1:].cpu(), torch.zeros(3))
    for tol, stops in ((1e-30, False), (1e30, True)):
        torch.mul(dgd, p, out=Apd)
        _call("spo_ma_dots", _ptr(p), _ptr(Apd), *[None] * 6, 1, P, _ptr(work), _ptr(st[1:]), _stream())
        torch.cuda.synchronize()
        x0, r0, p0, s0, Ap = (t.cpu().double() for t in (x, r, p, st, Apd))
        prod = p0 * Ap
        _check("vec", st[1:2], prod.sum().reshape(1), scale=float(prod.abs().sum()))
        _call("spo_ma_cg_update", _ptr(x), _ptr(r), _ptr(p), _ptr(Apd), P, tol, _ptr(work), _ptr(st), _stream())
        torch.cuda.synchronize()
        # the step from the kernel's own inputs (its fp32 p.Ap included); scales: the size of the terms that cancel
        alpha = s0[0] / (s0[1] + 1e-8)
        x64, r64 = x0 + alpha * p0, r0 - alpha * Ap
        _check("vec", x, x64, scale=float(x0.abs().max() + (alpha * p0).abs().max()))
        _check("vec", r, r64, scale=float(r0.abs().max() + (alpha * Ap).abs().max()))
        rk = r.cpu().double()
        nr = (rk ** 2).sum()
        _check("vec", st[0:1], nr.reshape(1))
        _check("vec", st[2:3], (st[0].cpu().double() / s0[0]).reshape(1))
        assert float(st[3]) == (1.0 if stops else 0.0)
        if stops:
            assert torch.equal(p.cpu().double(), p0)          # a stopped solve does not take the new direction
        else:
            beta = st[2].cpu().double()
            _check("vec", p, rk + beta * p0, scale=float(rk.abs().max() + (beta * p0).abs().max()))
        for t in (x, r, p):
            assert bool((t.cpu()[pad] == 0).all())
    frozen = [t.clone() for t in (x, r, p, st)]
    _call("spo_ma_cg_update", _ptr(x), _ptr(r), _ptr(p), _ptr(Apd), P, 1e30, _ptr(work), _ptr(st), _stream())
    torch.cuda.synchronize()
    assert all(torch.equal(a_, b_) for a_, b_ in zip((x, r, p, st), frozen))
    # ---- step direction ----
    xg, xb = vec(), vec()
    xgd, xbd, xs = xg.to(dev), xb.to(dev), torch.empty(P, device=dev)
    for use_a, c, nu in ((1, 0.7, 0.3), (0, 0.0, 1.9)):
        _call("spo_ma_step_dir", _ptr(xgd) if use_a else None, _ptr(xbd), c, nu, use_a, _ptr(xs), P, _stream())
        torch.cuda.synchronize()
        want = c * (xg.double() + nu * xb.double()) if use_a else nu * xb.double()
        _check("vec", xs, want)
        assert bool((xs.cpu()[pad] == 0).all())
    # ---- line-search trial: |x| above 0.5 (rescaled, written back) and below (untouched) ----
    old = vec()
    oldd = old.to(dev)
    for norm_target in (3.0, 0.2):
        xv = vec()
        xv = xv * (norm_target / float(xv.double().norm()))
        xd, xsq, out = xv.to(dev), torch.empty(1, device=dev), torch.empty(P, device=dev)
        _call("spo_ma_dots", _ptr(xd), _ptr(xd), *[None] * 6, 1, P, _ptr(work), _ptr(xsq), _stream())
        _call("spo_ma_ls_trial", _ptr(oldd), _ptr(xd), _ptr(xsq), 0.05, _ptr(out), P, _stream())
        torch.cuda.synchronize()
        nrm = float(xv.double().norm())
        x64 = xv.double() * 0.5 / nrm if nrm > 0.5 else xv.double()
        if nrm > 0.5:
            _check("vec", xd, x64)
        else:
            assert torch.equal(xd.cpu(), xv)
        _check("vec", out, old.double() - 0.05 * x64, scale=float(old.abs().max()) + 0.05 * float(x64.abs().max()))
        assert bool((out.cpu()[pad] == 0).all())


# ============================================================ GPU: whole steps ============================================================
# (name, N, D, DS, A, H, layer_N, cfg changes): the MAMuJoCo section of the reference's MACPO yaml (layer_N 1, hidden 128, gamma 0.99,
# entropy_coef 0.01), H = 384 with 32 action dimensions, one row with obs 2 and one action dimension, config 5's layer shape
STEPS = [("mamujoco", 1000, 18, 36, 3, 128, 1, dict(gamma=0.99, entropy_coef=0.01)),
         ("h384_a32", 300, 66, 66, 32, 384, 2, dict(entropy_coef=0.01, huber_delta=1.0)),
         ("tiny", 1, 2, 2, 1, 128, 2, dict(entropy_coef=0.01)),
         ("config5", 4097, 398, 398, 20, 512, 2, dict(entropy_coef=0.01))]


def _step_setup(name, N, D, DS, A, H, layer_N, changes, dev):
    from safepo.common.ma_model import MultiAgentNets
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    sts = (_state(g, D, H, A, "actor", layer_N), _state(g, DS, H, A, "critic", layer_N), _state(g, DS, H, A, "critic", layer_N))
    cfg = dict(actor_lr=9e-5, critic_lr=5e-3, opti_eps=1e-5, weight_decay=0.0, clip_param=0.2, huber_delta=10.0, entropy_coef=0.0,
               max_grad_norm=10.0, cost_limit=25.0, gamma=0.96, lagrangian_coef_rate=1e-5, value_loss_coef=1.0, lamda_lagr=0.78,
               std_x_coef=1.0, std_y_coef=0.5)
    cfg.update(changes)
    s = _sample(g, N, D, DS, A, sts[0], layer_N, cfg["std_x_coef"], cfg["std_y_coef"])
    nets = MultiAgentNets(*sts, dev, layer_N=layer_N, std_x_coef=cfg["std_x_coef"], std_y_coef=cfg["std_y_coef"])
    return sts, cfg, s, nets, g


@pytest.mark.gpu
@pytest.mark.parametrize("case", STEPS, ids=[c[0] for c in STEPS])
def test_ppo_update_readout_vs_float64(case):
    """MultiAgentTrainer.ppo_update: the gradient of every parameter tensor before the clip (net.gflat), the eight returned
    values, lambda and the PopArt state against the float64 reference."""
    from safepo.common.ma_model import MultiAgentTrainer
    dev = _cuda()
    name, N, D, DS, A, H, layer_N, changes = case
    sts, cfg, s, nets, _ = _step_setup(*case, dev)
    tr = MultiAgentTrainer(nets, cfg)
    got = tr.ppo_update(s)
    torch.cuda.synchronize()
    want = ref_ppo_update(sts, s, cfg, torch.float64, layer_N)
    for net, wg in zip((nets.actor, nets.critic, nets.cost_critic), want["grads"]):
        for k, w in wg.items():
            _check("step_grad", net.g[k], w)
    names = ("value_loss", "critic_grad_norm", "policy_loss", "dist_entropy", "actor_grad_norm", "imp_weights", "cost_loss", "cost_grad_norm")
    adv = s["adv_targ"].double() - cfg["lamda_lagr"] * s["cost_adv_targ"].double()
    for k, v in zip(names, got):
        w = want["out"][k]
        scale = float((s["factor"].double() * want["imp"] * adv).abs().mean()) if k == "policy_loss" else None
        _check("step_scalar", v.reshape(-1), torch.as_tensor(w).reshape(-1), scale=scale)
    _check("step_scalar", tr.lamda_lagr, torch.as_tensor(want["lamda"]).reshape(1), scale=cfg["lamda_lagr"])
    _check("step_scalar", tr.popart_state, want["popart"].state())


@pytest.mark.gpu
@pytest.mark.parametrize("case", STEPS, ids=[c[0] for c in STEPS])
def test_macpo_fvp_and_surrogate_grad_readout_vs_float64(case):
    """MACPOTrainer.fvp and .surrogate_grad per tensor against float64 double backprop / autograd of the reference's KL and
    ratio surrogates."""
    from safepo.common.ma_model import MACPOTrainer, _tangent_views
    dev = _cuda()
    name, N, D, DS, A, H, layer_N, changes = case
    sts, cfg, s, nets, g = _step_setup(*case, dev)
    tr = MACPOTrainer(nets, dict(MA_DEFAULT_CFG(), **cfg, layer_N=layer_N, hidden_size=H))
    net = nets.actor
    obs = s["obs"].to(dev).contiguous()
    mean_old = tr.actor_forward(obs)
    v = torch.zeros(net.flat.numel())
    vt = _tangent_views(net, v)
    for k in vt:
        vt[k].copy_(0.1 * torch.randn(vt[k].shape, generator=g))
    vd, out = v.to(dev), torch.empty(net.flat.numel(), device=dev)
    tr.fvp(vd, out)
    torch.cuda.synchronize()
    p64 = {k: t.double().requires_grad_(True) for k, t in sts[0].items()}
    v64 = torch.cat([vt[k].reshape(-1) for k in sts[0]]).double()
    want = ref_fvp(p64, s["obs"].double(), v64, layer_N, cfg["std_x_coef"], cfg["std_y_coef"])
    got = _tangent_views(net, out.cpu())
    i = 0
    for k, t in sts[0].items():
        _check("step_fvp", got[k], want[i:i + t.numel()].view(t.shape))
        i += t.numel()
    pad = torch.ones(net.flat.numel(), dtype=torch.bool)
    for k in vt:
        pad[(net.p[k].data_ptr() - net.flat.data_ptr()) // 4:][:net.p[k].numel()] = False
    assert bool((out.cpu()[pad] == 0).all())
    # ratio surrogates
    dd = {k: torch.as_tensor(t, dtype=torch.float32).to(dev).contiguous() for k, t in s.items()}
    dist = actor_dist(p64, s["obs"].double(), layer_N, cfg["std_x_coef"], cfg["std_y_coef"])
    rl, cl, ratio = ratio_surrogates(dist.log_prob(s["actions"].double()), s["old_action_log_probs"].double(), s["factor"].double(),
                                     s["adv_targ"].double(), s["cost_adv_targ"].double())
    lbuf = torch.zeros(32, device=dev)
    for sign, advk, L in ((-1.0, "adv_targ", rl), (1.0, "cost_adv_targ", cl)):
        gv = torch.zeros_like(net.flat)
        tr.surrogate_grad(mean_old, dd["actions"], dd["old_action_log_probs"], dd[advk].reshape(-1), dd["factor"].reshape(-1), sign, lbuf, gv)
        torch.cuda.synchronize()
        wg = torch.autograd.grad(L, list(p64.values()), retain_graph=True)
        views = _tangent_views(net, gv.cpu())
        for (k, _), w in zip(sts[0].items(), wg):
            _check("step_surr", views[k], w)
        _check("step_surr", lbuf[0:1], L.detach().reshape(1),
               scale=float((ratio.detach() * s["factor"].double() * s[advk].double()).abs().mean()))
        assert bool((gv.cpu()[pad] == 0).all())
