"""Multi-agent (MAPPO-Lag) networks on the device (SURVEY section 8f rank 3).

``MultiAgentNets`` holds the weights of one agent's actor, reward critic and cost critic under the reference's own
``state_dict`` names (safepo/common/model.py:172-363: ``base.feature_norm``, ``base.mlp.fc1``, ``base.mlp.fc2.{i}``,
``act.action_out`` / ``v_out``) and evaluates ``MAPPO_L_Policy.get_actions`` (safepo/multi_agent/mappolag.py:69-82) with
libspo kernels: one ``spo_ma_mlp_layer`` launch per hidden layer and one ``spo_ma_head`` launch per net.

The trainers share one base (``_AgentTrainer``): training forward with the activations kept, the backward pass layer by
layer (``spo_ma_ln_elu_bwd``, ``spo_ma_gemm_tn``, ``spo_ma_gemm_nn``), ``clip_grad_norm_`` + Adam on the packed parameters
(``spo_ma_clip_adam``), the PopArt critic update with its clipped-Huber loss, the sample decoding and the resumable state --
no host synchronisation inside an update, no CPU path.  Each net's parameters live in one packed fp32 buffer;
``net.p[name]`` are views into it.  Each algorithm adds its own update on top:

``MultiAgentTrainer`` is the device side of ``MAPPO_L_Trainer.ppo_update`` (mappolag.py:135-199) for one agent: the
clipped-surrogate loss head and the Lagrange-multiplier step.

``MACPOTrainer`` is the device side of ``MACPO_Trainer.trpo_update`` / ``train`` (safepo/multi_agent/macpo.py:96-415): the
actor's trust-region step (spo_ma_trust.cu).

``MAPPOTrainer`` / ``HAPPOTrainer`` are ``MAPPO_Trainer`` / ``HAPPO_Trainer`` (safepo/multi_agent/mappo.py:96-186,
happo.py:96-194) on a two-net ``MultiAgentNets``: the loss heads of spo_ma_ppo.cu (per-dimension or product ratio, active
masks)."""
from __future__ import annotations

import os

import torch

from safepo import _lib as L


def _launch(name, *args):
    L.check(getattr(L.lib(), name)(*args), name)


class _Net:
    def __init__(self, state, device, layer_N):
        # one packed buffer per net (every tensor starts on a 16-byte boundary), parameters as views: the update kernels
        # run over the whole buffer, the layer kernels over the views
        offs, total = {}, 0
        for k, v in state.items():
            offs[k] = total
            total += (v.numel() + 3) // 4 * 4
        self.flat = torch.zeros(total, dtype=torch.float32, device=device)
        self.gflat = torch.zeros(total, dtype=torch.float32, device=device)      # gradients of the last update (before the clip)
        self.exp_avg = torch.zeros(total, dtype=torch.float32, device=device)
        self.exp_avg_sq = torch.zeros(total, dtype=torch.float32, device=device)
        self.p, self.g = {}, {}
        for k, v in state.items():
            sl = slice(offs[k], offs[k] + v.numel())
            self.p[k] = self.flat[sl].view(v.shape)
            self.g[k] = self.gflat[sl].view(v.shape)
            self.p[k].copy_(v.detach().to(device=device, dtype=torch.float32))
        self.layer_N = layer_N
        self.H = self.p["base.mlp.fc1.0.weight"].shape[0]
        self.D = self.p["base.mlp.fc1.0.weight"].shape[1]
        self.step = 0            # Adam step count
        # (weight, bias, ln weight, ln bias) names of the 1 + layer_N blocks
        self.blocks = [("base.mlp.fc1.0.weight", "base.mlp.fc1.0.bias", "base.mlp.fc1.2.weight", "base.mlp.fc1.2.bias")] + \
            [(f"base.mlp.fc2.{i}.0.weight", f"base.mlp.fc2.{i}.0.bias", f"base.mlp.fc2.{i}.2.weight", f"base.mlp.fc2.{i}.2.bias")
             for i in range(layer_N)]

    def state_dict(self):
        return {k: v.detach().clone() for k, v in self.p.items()}

    def check_state(self, state, what):
        """Raise SpoError naming the first key of ``state`` that is missing, extra, not a floating tensor or of the wrong
        shape (load_state_dict(strict=True) refuses the same)."""
        if not isinstance(state, dict):
            raise L.SpoError(f"{what}: a state dict expected, got {type(state).__name__}")
        for k in self.p:
            if k not in state:
                raise L.SpoError(f"{what}: missing key {k!r}")
        for k, v in state.items():
            if k not in self.p:
                raise L.SpoError(f"{what}: unexpected key {k!r}")
            if not (torch.is_tensor(v) and v.is_floating_point()):
                raise L.SpoError(f"{what}: {k!r} is not a floating-point tensor")
            if tuple(v.shape) != tuple(self.p[k].shape):
                raise L.SpoError(f"{what}: {k!r} has shape {tuple(v.shape)}, expected {tuple(self.p[k].shape)}")

    def load_state(self, state):
        """Copy a checked state dict into the packed buffer in place (the views and the optimiser buffers stay valid)."""
        for k, v in state.items():
            self.p[k].copy_(v.detach().to(dtype=torch.float32))

    def cpu_state_dict(self):
        """The parameters as separate fp32 CPU tensors (not views of the packed buffer, so that torch.save writes each
        tensor alone), in the reference's names."""
        return {k: v.detach().cpu().clone() for k, v in self.p.items()}

    def features(self, x, work):
        """MLPBase.forward: feature_norm folded into the first layer's launch."""
        p, n = self.p, x.shape[0]
        a, b = work
        w, bb, lw, lb = self.blocks[0]
        _launch("spo_ma_mlp_layer", L.ptr(x), n, self.D, L.ptr(p[w]), L.ptr(p[bb]), L.ptr(p[lw]), L.ptr(p[lb]), self.H,
                L.ptr(p["base.feature_norm.weight"]), L.ptr(p["base.feature_norm.bias"]), L.ptr(a), L.stream())
        for w, bb, lw, lb in self.blocks[1:]:
            _launch("spo_ma_mlp_layer", L.ptr(a), n, self.H, L.ptr(p[w]), L.ptr(p[bb]), L.ptr(p[lw]), L.ptr(p[lb]), self.H, None, None,
                    L.ptr(b), L.stream())
            a, b = b, a
        return a


class MultiAgentNets:
    def __init__(self, actor_state, critic_state, cost_critic_state=None, device="cuda", layer_N=2, std_x_coef=1.0, std_y_coef=0.5):
        """``cost_critic_state=None``: the two nets of MAPPO_Policy / HAPPO_Policy (mappo.py:46-62); ``cost_critic`` is then None."""
        device = torch.device(device)
        self._require_cuda(device)
        self.device = device
        self.actor = _Net(actor_state, device, layer_N)
        self.critic = _Net(critic_state, device, layer_N)
        self.cost_critic = None if cost_critic_state is None else _Net(cost_critic_state, device, layer_N)
        self.act_dim = self.actor.p["act.action_out.fc_mean.weight"].shape[0]
        self.std_x_coef, self.std_y_coef = float(std_x_coef), float(std_y_coef)
        self._work = {}

    @staticmethod
    def _require_cuda(device):
        if device.type != "cuda":
            raise L.SpoError("MultiAgentNets runs on a CUDA device only (no CPU fallback)")

    def _buffers(self, n, H):
        key = (n, H)
        if key not in self._work:
            self._work[key] = (torch.empty(n, H, dtype=torch.float32, device=self.device), torch.empty(n, H, dtype=torch.float32, device=self.device))
        return self._work[key]

    def head(self, net, feat, out, eps=None, logp=None):
        """The ``spo_ma_head`` launch on the features [n, H] of ``net``: a critic's values [n, 1], or the actor's actions
        [n, A] (the means without ``eps``, mean + std * eps with it) and, given ``logp``, their per-dimension log-probabilities."""
        if net is self.actor:
            w, b, O, ls, x, y = (net.p["act.action_out.fc_mean.weight"], net.p["act.action_out.fc_mean.bias"], self.act_dim,
                                 net.p["act.action_out.log_std"], self.std_x_coef, self.std_y_coef)
        else:
            w, b, O, ls, x, y = net.p["v_out.weight"], net.p["v_out.bias"], 1, None, 1.0, 1.0
        _launch("spo_ma_head", L.ptr(feat), feat.shape[0], net.H, L.ptr(w), L.ptr(b), O, L.ptr(ls), x, y, L.ptr(eps), L.ptr(out), L.ptr(logp),
                L.stream())
        return out

    def value(self, net, cent_obs):
        """The values [N, 1] of the critic ``net`` (``critic`` or ``cost_critic``) on ``cent_obs``."""
        n = cent_obs.shape[0]
        feat = net.features(cent_obs, self._buffers(n, net.H))
        return self.head(net, feat, torch.empty(n, 1, dtype=torch.float32, device=self.device))

    def get_actions(self, cent_obs, obs, eps=None, deterministic=False):
        """(values [N,1], actions [N,A], action_log_probs [N,A], cost_preds [N,1]) like MAPPO_L_Policy.get_actions (cost_preds
        None without a cost critic).  ``eps`` [N,A]: the standard-normal draws to use (torch.randn on the device when omitted and
        not deterministic)."""
        for t in (cent_obs, obs):
            if not (t.device.type == self.device.type and t.dtype == torch.float32 and t.is_contiguous()):   # self.device is CUDA (constructor)
                raise L.SpoError("MultiAgentNets needs contiguous fp32 CUDA tensors")
        n, A, net = obs.shape[0], self.act_dim, self.actor
        feat = net.features(obs, self._buffers(n, net.H))
        if deterministic:
            eps = None
        elif eps is None:
            eps = torch.randn(n, A, dtype=torch.float32, device=self.device)
        actions = torch.empty(n, A, dtype=torch.float32, device=self.device)
        logp = torch.empty(n, A, dtype=torch.float32, device=self.device)
        self.head(net, feat, actions, eps, logp)
        cost_preds = None if self.cost_critic is None else self.value(self.cost_critic, cent_obs)
        return self.value(self.critic, cent_obs), actions, logp, cost_preds

    def act(self, obs):
        """The deterministic actions [N, A] (the means) of MAPPO_L_Policy.act(..., deterministic=True) (mappolag.py:107-109):
        the actor alone, no critic."""
        if not (obs.device.type == self.device.type and obs.dtype == torch.float32 and obs.is_contiguous()):
            raise L.SpoError("MultiAgentNets needs contiguous fp32 CUDA tensors")
        n, A, net = obs.shape[0], self.act_dim, self.actor
        feat = net.features(obs, self._buffers(n, net.H))
        return self.head(net, feat, torch.empty(n, A, dtype=torch.float32, device=self.device))

    # ---- checkpoints in the reference's format (Runner.save / restore, mappolag.py:506-518) ----
    @staticmethod
    def checkpoint_paths(directory, agent_id):
        return (os.path.join(directory, f"actor_agent{agent_id}.pt"), os.path.join(directory, f"critic_agent{agent_id}.pt"))

    def save(self, directory, agent_id):
        """Write ``actor_agent{i}.pt`` and ``critic_agent{i}.pt``: CPU fp32 state dicts under the reference's keys, which the
        reference's Runner.restore loads as they are.  Like the reference, the cost critic is not written."""
        os.makedirs(directory, exist_ok=True)
        for net, path in zip((self.actor, self.critic), self.checkpoint_paths(directory, agent_id)):
            torch.save(net.cpu_state_dict(), path)

    def load(self, directory, agent_id):
        """Read ``actor_agent{i}.pt`` / ``critic_agent{i}.pt`` (written by ``save`` or by the reference) into the packed
        buffers in place.  Both files are checked before either is copied: a missing file, a missing or extra key or a wrong
        shape raises SpoError naming it.  The cost critic, which the reference does not save, keeps its weights."""
        states = []
        for net, path in zip((self.actor, self.critic), self.checkpoint_paths(directory, agent_id)):
            if not os.path.isfile(path):
                raise L.SpoError(f"no checkpoint {path}")
            state = torch.load(path, map_location="cpu", weights_only=True)
            net.check_state(state, path)
            states.append(state)
        for net, state in zip((self.actor, self.critic), states):
            net.load_state(state)


    def evaluate_actions(self, obs, actions):
        """Per-dimension log-probabilities of given actions under the current actor (MultiAgentActor.evaluate_actions,
        model.py:270-296 -> act.py:62-77), as the runner needs them for the cross-agent factor (mappolag.py:474-497): the mean
        from the forward kernels, then Normal.log_prob's own formula element-wise on the device."""
        n, A, net = obs.shape[0], self.act_dim, self.actor
        feat = net.features(obs, self._buffers(n, net.H))
        mean = self.head(net, feat, torch.empty(n, A, dtype=torch.float32, device=self.device))
        std = torch.sigmoid(net.p["act.action_out.log_std"] / self.std_x_coef) * self.std_y_coef
        return -((actions - mean) ** 2) / (2 * std ** 2) - std.log() - _LOG_SQRT_2PI


_LOG_SQRT_2PI = 0.9189385332046727      # math.log(math.sqrt(2 * math.pi)), torch.distributions.Normal.log_prob

# the 18 positions of the sample tuple MAPPO_L_Trainer.ppo_update unpacks (mappolag.py:137-141)
_SAMPLE_KEYS = ("share_obs", "obs", "rnn_states", "rnn_states_critic", "actions", "value_preds", "returns", "masks", "active_masks",
                "old_action_log_probs", "adv_targ", "available_actions", "factor", "cost_preds", "cost_returns", "rnn_states_cost",
                "cost_adv_targ", "aver_episode_costs")


# the 13 positions of the sample tuple MAPPO_Trainer / HAPPO_Trainer.ppo_update unpack (mappo.py:120-122, happo.py:125-127;
# buffer.py:465)
_PPO_SAMPLE_KEYS = ("share_obs", "obs", "rnn_states", "rnn_states_critic", "actions", "value_preds", "returns", "masks", "active_masks",
                    "old_action_log_probs", "adv_targ", "available_actions", "factor")


def _standardised_advantages(returns, preds, mean, sd):
    """The advantages of MACPO, MAPPO and HAPPO (macpo.py:384-388, mappo.py:165-170, happo.py:173-178): returns - denormalised
    predictions, standardised by the mean and unbiased std + 1e-5 over every entry (no NaN masking, unlike MAPPO-Lag's)."""
    adv = returns[:-1] - (preds[:-1] * sd + mean)
    return (adv - adv.mean()) / (adv.std() + 1e-5)


class _AgentTrainer:
    """What every multi-agent trainer does the same way for one agent around ``MultiAgentNets``: the training forward, the
    backward chain, clip + Adam, the PopArt critic update, the sample decoding and the resumable state.  The updates themselves
    are the subclasses'.  ``cfg`` carries the reference's keys: actor_lr, critic_lr, opti_eps, weight_decay, clip_param,
    huber_delta, max_grad_norm, value_loss_coef, and the algorithm's own."""

    SAMPLE_KEYS = _SAMPLE_KEYS      # the positions of the reference's sample tuple
    USES_FACTOR = True              # the actor's loss takes the cross-agent factor

    def __init__(self, nets: MultiAgentNets, cfg):
        self.nets, self.cfg, self.device = nets, dict(cfg), nets.device
        dev = self.device
        # train_state_agent{i}.pt holds a Lagrange multiplier for every algorithm; only MAPPO-Lag's update moves it
        self.lamda_lagr = torch.full((1,), float(cfg.get("lamda_lagr", 0.0)), dtype=torch.float32, device=dev)
        self.popart_state = torch.zeros(3, dtype=torch.float32, device=dev)     # running_mean, running_mean_sq, debiasing_term
        self.popart_beta, self.popart_eps = 0.99999, 1e-5                      # popart.py:48
        self._adam_work = torch.empty(1024, dtype=torch.float32, device=dev)
        self._bufs = {}

    # ---- workspace ----
    def _ws(self, n, net):
        key = (n, net.D, net.H, net.layer_N)
        if key not in self._bufs:
            dev, H, D, nl = self.device, net.H, net.D, 1 + net.layer_N
            A = self.nets.act_dim
            f = dict(dtype=torch.float32, device=dev)
            nb32, nb256 = (n + 31) // 32, (n + 255) // 256
            wmax = max(H * max(H, D), A * H)
            self._bufs[key] = dict(
                xn=torch.empty(n, D, **f), pre=[torch.empty(n, H, **f) for _ in range(nl)], out=[torch.empty(n, H, **f) for _ in range(nl)],
                dy=torch.empty(n, max(H, D), **f), dy2=torch.empty(n, max(H, D), **f), dz=torch.empty(n, H, **f),
                part=torch.empty(max(nb32 * 3 * H, nb32 * 2 * D, nb32 * 66, nb256 * 2, 32 * wmax), **f),
                dmean=torch.empty(n, A, **f), v=torch.empty(n, 1, **f), dv=torch.empty(n, **f), rn_c=torch.empty(n, **f), rn_o=torch.empty(n, **f))
        return self._bufs[key]

    # ---- pieces ----
    def _forward_train(self, net, x, ws):
        p, n = net.p, x.shape[0]
        w, bb, lw, lb = net.blocks[0]
        _launch("spo_ma_mlp_layer_train", L.ptr(x), n, net.D, L.ptr(p[w]), L.ptr(p[bb]), L.ptr(p[lw]), L.ptr(p[lb]), net.H,
                L.ptr(p["base.feature_norm.weight"]), L.ptr(p["base.feature_norm.bias"]), L.ptr(ws["out"][0]), L.ptr(ws["pre"][0]),
                L.ptr(ws["xn"]), L.stream())
        for i, (w, bb, lw, lb) in enumerate(net.blocks[1:], start=1):
            _launch("spo_ma_mlp_layer_train", L.ptr(ws["out"][i - 1]), n, net.H, L.ptr(p[w]), L.ptr(p[bb]), L.ptr(p[lw]), L.ptr(p[lb]), net.H,
                    None, None, L.ptr(ws["out"][i]), L.ptr(ws["pre"][i]), None, L.stream())
        return ws["out"][-1]

    def _gemm_tn(self, A_, B_, out, R, M, N, ws):
        """out[M][N] = A_[R][M]^T B_[R][N] (sum over the R rows in slices, partials reduced in order)."""
        tiles = ((M + 127) // 128) * ((N + 63) // 64)            # 128 x 64 output tiles, >= 2 CTAs per SM wanted
        slices = max(1, min(32, (296 + tiles - 1) // tiles, R // 256))
        while slices > 1 and (slices - 1) * (((R + slices - 1) // slices + 31) // 32 * 32) >= R:   # no empty slice (32-row chunks)
            slices -= 1
        _launch("spo_ma_gemm_tn", L.ptr(A_), L.ptr(B_), L.ptr(ws["part"]), R, M, N, slices, L.stream())
        _launch("spo_ma_partial_reduce", L.ptr(ws["part"]), slices, M * N, 1, M * N, L.ptr(out), None, None, 1.0, L.stream())

    def _backward(self, net, x, ws, dfeat):
        """Gradients of every block and of the input LayerNorm from dfeat = d loss / d features (in ws['dy'])."""
        p, g, n, H = net.p, net.g, x.shape[0], net.H
        nb32 = (n + 31) // 32
        dy, dy2 = dfeat, (ws["dy2"] if dfeat is ws["dy"] else ws["dy"])
        for i in reversed(range(len(net.blocks))):
            w, bb, lw, lb = net.blocks[i]
            _launch("spo_ma_ln_elu_bwd", L.ptr(dy), L.ptr(ws["pre"][i]), L.ptr(p[lw]), n, H, L.ptr(ws["dz"]), L.ptr(ws["part"]), L.stream())
            _launch("spo_ma_partial_reduce", L.ptr(ws["part"]), nb32, 3 * H, 3, H, L.ptr(g[lw]), L.ptr(g[lb]), L.ptr(g[bb]), 1.0, L.stream())
            inp, K = (ws["out"][i - 1], H) if i > 0 else (ws["xn"], net.D)
            self._gemm_tn(ws["dz"], inp, g[w], n, H, K, ws)
            _launch("spo_ma_gemm_nn", L.ptr(ws["dz"]), L.ptr(p[w]), L.ptr(dy2), n, K, H, L.stream())
            dy, dy2 = dy2, dy
        _launch("spo_ma_ln_in_bwd", L.ptr(dy), L.ptr(x), n, net.D, L.ptr(ws["part"]), L.stream())
        _launch("spo_ma_partial_reduce", L.ptr(ws["part"]), nb32, 2 * net.D, 2, net.D, L.ptr(g["base.feature_norm.weight"]),
                L.ptr(g["base.feature_norm.bias"]), None, 1.0, L.stream())

    def _vjp_from_mean(self, net, obs, feat, ws):
        """Gradients of every actor parameter below the mean layer's bias from ws['dmean'] = d loss / d means."""
        n, H, A = obs.shape[0], net.H, self.nets.act_dim
        wm = net.p["act.action_out.fc_mean.weight"]
        self._gemm_tn(ws["dmean"], feat, net.g["act.action_out.fc_mean.weight"], n, A, H, ws)
        _launch("spo_ma_gemm_nn", L.ptr(ws["dmean"]), L.ptr(wm), L.ptr(ws["dy"]), n, H, A, L.stream())
        self._backward(net, obs, ws, ws["dy"])

    def _clip_adam(self, net, lr):
        c = self.cfg
        net.step += 1
        norm = torch.empty(2, dtype=torch.float32, device=self.device)
        _launch("spo_ma_clip_adam", L.ptr(net.flat), L.ptr(net.gflat), L.ptr(net.exp_avg), L.ptr(net.exp_avg_sq), net.flat.numel(),
                float(c["max_grad_norm"]), float(lr), 0.9, 0.999, float(c["opti_eps"]), float(c["weight_decay"]), net.step,
                L.ptr(self._adam_work), L.ptr(norm), L.stream())
        return norm[0]

    def _critic_update(self, net, share_obs, value_preds, returns, active_masks=None, mask_sum=None):
        """cal_value_loss (mappolag.py:121-133) + the critic's optimiser step (:174-186); returns (loss, grad norm).  With
        ``active_masks`` [n] and their device sum ``mask_sum`` the rows are weighted m_r / sum m (happo.py:117-118)."""
        c, n, H = self.cfg, share_obs.shape[0], net.H
        ws = self._ws(n, net)
        feat = self._forward_train(net, share_obs, ws)
        self.nets.head(net, feat, ws["v"])
        # the reference normalises the returns twice, UPDATING the shared statistics both times: first for the clipped error
        for dst in (ws["rn_c"], ws["rn_o"]):
            _launch("spo_ma_popart_normalize", L.ptr(returns), n, L.ptr(self.popart_state), self.popart_beta, self.popart_eps, L.ptr(dst), L.stream())
        nb256 = (n + 255) // 256
        if active_masks is None:
            _launch("spo_ma_value_loss", L.ptr(ws["v"]), L.ptr(value_preds), L.ptr(ws["rn_c"]), L.ptr(ws["rn_o"]), n, float(c["clip_param"]),
                    float(c["huber_delta"]), float(c["value_loss_coef"]) / n, L.ptr(ws["dv"]), L.ptr(ws["part"]), L.stream())
        else:
            _launch("spo_ma_value_loss_masked", L.ptr(ws["v"]), L.ptr(value_preds), L.ptr(ws["rn_c"]), L.ptr(ws["rn_o"]), L.ptr(active_masks),
                    L.ptr(mask_sum), n, float(c["clip_param"]), float(c["huber_delta"]), float(c["value_loss_coef"]), L.ptr(ws["dv"]),
                    L.ptr(ws["part"]), L.stream())
        loss = torch.empty(1, dtype=torch.float32, device=self.device)
        _launch("spo_ma_partial_reduce", L.ptr(ws["part"]), nb256, 2, 1, 1, L.ptr(loss), None, None, 1.0 / n if active_masks is None else 1.0,
                L.stream())
        _launch("spo_ma_partial_reduce", L.ptr(ws["part"]), nb256, 2, 2, 1, None, L.ptr(net.g["v_out.bias"]), None, 1.0, L.stream())
        self._gemm_tn(ws["dv"], feat, net.g["v_out.weight"], n, 1, H, ws)
        _launch("spo_ma_gemm_nn", L.ptr(ws["dv"]), L.ptr(net.p["v_out.weight"]), L.ptr(ws["dy"]), n, H, 1, L.stream())
        self._backward(net, share_obs, ws, ws["dy"])
        return loss[0], self._clip_adam(net, c["critic_lr"])

    def _device_sample(self, sample):
        """The fields of one sample (a dict with the buffer's keys, or the reference's tuple in the order of ``SAMPLE_KEYS``)
        as contiguous fp32 device tensors: obs, share_obs, actions, old log-probs [n, cols]; value_preds, returns, adv_targ,
        factor, active_masks, cost_preds, cost_returns, cost_adv_targ [n]; then aver_episode_costs as the sample holds it (only
        its mean is used).  What the trainer does not read comes back None: the factor without ``USES_FACTOR``, the cost fields
        when ``SAMPLE_KEYS`` has none, the active masks when the sample has none or the config turns no mask flag on."""
        if not isinstance(sample, dict):
            sample = {k: v for k, v in zip(self.SAMPLE_KEYS, sample)}
        dev, c = self.device, self.cfg

        def dv_(key, cols=None):
            t = torch.as_tensor(sample[key], dtype=torch.float32).to(dev).contiguous()
            return t.reshape(t.shape[0], -1) if cols is None else t.reshape(-1)
        masks = (c.get("use_policy_active_masks") or c.get("use_value_active_masks")) and sample.get("active_masks") is not None
        out = (dv_("obs"), dv_("share_obs"), dv_("actions"), dv_("old_action_log_probs"), dv_("value_preds", 1), dv_("returns", 1),
               dv_("adv_targ", 1), dv_("factor", 1) if self.USES_FACTOR else None, dv_("active_masks", 1) if masks else None)
        if "cost_adv_targ" not in self.SAMPLE_KEYS:
            return out + (None, None, None, None)
        return out + (dv_("cost_preds", 1), dv_("cost_returns", 1), dv_("cost_adv_targ", 1), sample["aver_episode_costs"])

    # ---- resumable state (train_state_agent{i}.pt, an extension: the reference saves none) ----
    def _named_nets(self):
        nets = self.nets
        return [(k, n) for k, n in (("actor", nets.actor), ("critic", nets.critic), ("cost_critic", nets.cost_critic)) if n is not None]

    def train_state(self):
        """Everything the trainer carries from one iteration to the next, as CPU tensors: per net the Adam moments (under the
        parameter names) and step count, the PopArt state and the Lagrange multiplier.  (MACPOTrainer carries nothing more:
        its trust-region step starts from the current actor every iteration.)"""
        nets = {}
        for name, net in self._named_nets():
            nets[name] = dict(step=int(net.step),
                              exp_avg={k: v.detach().cpu().clone() for k, v in _tangent_views(net, net.exp_avg).items()},
                              exp_avg_sq={k: v.detach().cpu().clone() for k, v in _tangent_views(net, net.exp_avg_sq).items()})
        return dict(nets=nets, popart_state=self.popart_state.detach().cpu().clone(), lamda_lagr=self.lamda_lagr.detach().cpu().clone())

    def load_train_state(self, state, what="train state"):
        """Restore what ``train_state`` returned, in place; every field is checked before anything is copied (SpoError naming
        the first bad one)."""
        if not isinstance(state, dict) or not isinstance(state.get("nets"), dict):
            raise L.SpoError(f"{what}: not a training state")
        names = [k for k, _ in self._named_nets()]
        if sorted(state["nets"]) != sorted(names):
            raise L.SpoError(f"{what}: nets {sorted(state['nets'])}, expected {sorted(names)}")
        for name, net in self._named_nets():
            s = state["nets"][name]
            if not isinstance(s, dict) or not isinstance(s.get("step"), int):
                raise L.SpoError(f"{what}: {name} has no Adam step count")
            for m in ("exp_avg", "exp_avg_sq"):
                net.check_state(s.get(m), f"{what}: {name}.{m}")
        for k, n in (("popart_state", 3), ("lamda_lagr", 1)):
            v = state.get(k)
            if not (torch.is_tensor(v) and v.is_floating_point() and v.numel() == n):
                raise L.SpoError(f"{what}: {k!r} must be a floating-point tensor of {n} elements")
        for name, net in self._named_nets():
            s = state["nets"][name]
            net.step = s["step"]
            for m, buf in (("exp_avg", net.exp_avg), ("exp_avg_sq", net.exp_avg_sq)):
                views = _tangent_views(net, buf)
                for k, v in s[m].items():
                    views[k].copy_(v.to(dtype=torch.float32))
        self.popart_state.copy_(state["popart_state"].reshape(3).to(torch.float32))
        self.lamda_lagr.copy_(state["lamda_lagr"].reshape(1).to(torch.float32))

    # ---- PopArt statistics ----
    def popart_mean_sqrt_var(self):
        """(mean, sqrt(var)) of the PopArt normaliser as host floats (popart.py:64-74): one device -> host copy of 3 floats."""
        st = self.popart_state.cpu()
        den = st[2].clamp(min=self.popart_eps)
        mean, mean_sq = st[0] / den, st[1] / den
        var = (mean_sq - mean ** 2).clamp(min=1e-2)
        return float(mean), float(torch.sqrt(var))


class MultiAgentTrainer(_AgentTrainer):
    """``MAPPO_L_Trainer`` for one agent around ``MultiAgentNets`` (mappolag.py:115-199; MLP policy, no recurrence, clipped +
    Huber value loss with the shared PopArt normaliser).  ``cfg`` adds the reference's entropy_coef, cost_limit, gamma,
    lagrangian_coef_rate, lamda_lagr, learning_iters and use_policy_active_masks (the yaml's mamujoco section turns it on: the
    surrogate rows weighted m_r / sum m and the masked entropy, mappolag.py:167-170).  As in the reference, the Lagrange step
    and both value losses ignore the masks, so use_value_active_masks changes nothing here."""

    # ---- the update ----
    def ppo_update(self, sample):
        """One update on the whole sample (a dict with the oracle's keys, or the reference's 18-tuple).  Returns
        (value_loss, critic_grad_norm, policy_loss, dist_entropy, actor_grad_norm, imp_weights, cost_loss, cost_grad_norm) as device
        tensors, like mappolag.py:199."""
        dev, c, nets = self.device, self.cfg, self.nets
        (obs, share_obs, actions, old_logp, value_preds, returns, adv, factor, active, cost_preds, cost_returns, cost_adv,
         aver_costs) = self._device_sample(sample)
        n, A = obs.shape[0], nets.act_dim
        pol_masks = bool(c.get("use_policy_active_masks", False))
        if pol_masks and active is None:
            raise L.SpoError("use_policy_active_masks needs the sample's active_masks")
        aver_costs = torch.as_tensor(aver_costs, dtype=torch.float32).to(dev).contiguous().reshape(-1)
        if aver_costs.numel() != n:      # the reference only uses aver_episode_costs.mean() (mappolag.py:170); its buffer field is not [n]
            aver_costs = aver_costs.mean().expand(n).contiguous()

        # ---- actor: surrogate on the product of the per-dimension ratios, Lagrangian-mixed advantage ----
        net = nets.actor
        ws = self._ws(n, net)
        feat = self._forward_train(net, obs, ws)
        nb32 = (n + 31) // 32
        imp = torch.empty(n, 1, dtype=torch.float32, device=dev)
        wm, bm, ls = net.p["act.action_out.fc_mean.weight"], net.p["act.action_out.fc_mean.bias"], net.p["act.action_out.log_std"]
        if not pol_masks:
            _launch("spo_ma_actor_loss", L.ptr(feat), n, net.H, L.ptr(wm), L.ptr(bm), L.ptr(ls), A, L.ptr(actions), L.ptr(old_logp), L.ptr(adv),
                    L.ptr(cost_adv), L.ptr(factor), L.ptr(self.lamda_lagr), 1.0 - float(c["clip_param"]), 1.0 + float(c["clip_param"]),
                    nets.std_x_coef, nets.std_y_coef, L.ptr(ws["dmean"]), L.ptr(imp), L.ptr(ws["part"]), L.stream())
            scal = torch.empty(2, dtype=torch.float32, device=dev)
            _launch("spo_ma_actor_finalize", L.ptr(ws["part"]), nb32, n, L.ptr(ls), A, nets.std_x_coef, nets.std_y_coef, float(c["entropy_coef"]),
                    L.ptr(net.g["act.action_out.fc_mean.bias"]), L.ptr(net.g["act.action_out.log_std"]), L.ptr(scal), L.stream())
        else:
            # the same surrogate (product ratio x factor on the Lagrangian-mixed advantage) with the rows weighted m_r / sum m
            msum = active.sum().reshape(1)         # on the device: 0/1 floats, exact in any order
            _launch("spo_ma_ppo_actor_loss", L.ptr(feat), n, net.H, L.ptr(wm), L.ptr(bm), L.ptr(ls), A, L.ptr(actions), L.ptr(old_logp),
                    L.ptr(adv), L.ptr(cost_adv), L.ptr(self.lamda_lagr), L.ptr(factor), L.ptr(active), L.ptr(msum), L.MA_RATIO_PRODUCT,
                    1.0 - float(c["clip_param"]), 1.0 + float(c["clip_param"]), nets.std_x_coef, nets.std_y_coef, L.ptr(ws["dmean"]),
                    L.ptr(imp), L.ptr(ws["part"]), L.stream())
            scal = torch.empty(3, dtype=torch.float32, device=dev)
            _launch("spo_ma_ppo_actor_finalize", L.ptr(ws["part"]), nb32, n, L.ptr(msum), L.MA_RATIO_PRODUCT, L.ptr(ls), A, nets.std_x_coef,
                    nets.std_y_coef, float(c["entropy_coef"]), L.ptr(net.g["act.action_out.fc_mean.bias"]), L.ptr(net.g["act.action_out.log_std"]),
                    L.ptr(scal), L.stream())
        self._vjp_from_mean(net, obs, feat, ws)
        actor_grad_norm = self._clip_adam(net, c["actor_lr"])
        # ---- Lagrange multiplier (uses the importance weights of THIS update, mappolag.py:169-172) ----
        _launch("spo_ma_lagrange_step", L.ptr(imp), L.ptr(cost_adv), L.ptr(aver_costs), n, float(c["cost_limit"]), float(c["gamma"]),
                float(c["lagrangian_coef_rate"]), L.ptr(self.lamda_lagr), L.stream())
        # ---- critics ----
        value_loss, critic_grad_norm = self._critic_update(nets.critic, share_obs, value_preds, returns)
        cost_loss, cost_grad_norm = self._critic_update(nets.cost_critic, share_obs, cost_preds, cost_returns)
        return value_loss, critic_grad_norm, scal[0], scal[1], actor_grad_norm, imp, cost_loss, cost_grad_norm

    # ---- MAPPO_L_Trainer.train (mappolag.py:200-234) ----
    def train(self, buf, perms=None):
        """learning_iters whole-batch updates on a SeparatedReplayBuffer: advantages = returns - denormalised predictions,
        standardised by the mean / unbiased std over the entries (the reference writes NaN into inactive entries and then
        takes torch.mean, so a buffer with any inactive entry yields NaN advantages there too -- reproduced).  With
        use_policy_active_masks this means: as long as the agent was active at every step of the buffer, all masks are 1, the
        surrogate is the plain mean and only the entropy changes form (the masked entropy sums over the action dimensions);
        once the agent finished alone at some step, every advantage is NaN and so is the update, as in the reference.  ``perms``: the row orders to use (one per iteration; torch.randperm on the
        device when omitted)."""
        mean, sd = self.popart_mean_sqrt_var()

        def standardise(ret, pred):
            adv = ret[:-1] - (pred[:-1] * sd + mean)
            copy = adv.clone()
            copy[buf.active_masks[:-1] == 0.0] = float("nan")
            return (adv - torch.mean(copy)) / (torch.std(copy) + 1e-8)
        advantages = standardise(buf.returns, buf.value_preds)
        cost_adv = standardise(buf.cost_returns, buf.cost_preds)
        out = None
        for it in range(int(self.cfg["learning_iters"])):
            perm = None if perms is None else perms[it]
            out = self.ppo_update(buf.whole_batch_sample(advantages, cost_adv, perm))
        return out


class _TwoNetPPOTrainer(_AgentTrainer):
    """The update shared by ``MAPPO_Trainer`` and ``HAPPO_Trainer`` (mappo.py:96-186, happo.py:96-194) for one agent around a
    two-net ``MultiAgentNets`` (actor + reward critic): the loss head of ``spo_ma_ppo_actor_loss`` /
    ``spo_ma_ppo_actor_finalize`` and, where the algorithm honours ``use_value_active_masks``, the critic update with
    ``spo_ma_value_loss_masked``.  ``cfg`` carries the yaml's keys:
    actor_lr, critic_lr, opti_eps, weight_decay, clip_param, huber_delta, entropy_coef, max_grad_norm, value_loss_coef,
    learning_iters, use_policy_active_masks, use_value_active_masks."""

    SAMPLE_KEYS = _PPO_SAMPLE_KEYS
    RATIO_MODE = L.MA_RATIO_PRODUCT
    HONOURS_VALUE_MASKS = True

    def __init__(self, nets: MultiAgentNets, cfg):
        super().__init__(nets, cfg)
        self.last_ratio = None       # mean importance weight of the last update (the logged Misc/Ratio), a device scalar

    def ppo_update(self, sample):
        """One update on the whole sample (a dict with the buffer's keys, or the reference's 13-tuple).  Returns (value_loss,
        critic_grad_norm, policy_loss, dist_entropy, actor_grad_norm, imp_weights) as device tensors, like mappo.py:163 /
        happo.py:171: imp_weights is [n, 1] for the product ratio, [n, A] per dimension.  No host synchronisation."""
        dev, c, nets = self.device, self.cfg, self.nets
        obs, share_obs, actions, old_logp, value_preds, returns, adv, factor, active, *_ = self._device_sample(sample)
        n, A = obs.shape[0], nets.act_dim
        pol_masks = bool(c.get("use_policy_active_masks", False))
        val_masks = bool(c.get("use_value_active_masks", False)) and self.HONOURS_VALUE_MASKS
        if (pol_masks or val_masks) and active is None:
            raise L.SpoError("use_policy_active_masks / use_value_active_masks need the sample's active_masks")
        msum = active.sum().reshape(1) if (pol_masks or val_masks) else None      # on the device: 0/1 floats, exact in any order

        # ---- actor ----
        net = nets.actor
        ws = self._ws(n, net)
        feat = self._forward_train(net, obs, ws)
        nb32 = (n + 31) // 32
        mode = self.RATIO_MODE
        imp = torch.empty(n, A if mode == L.MA_RATIO_PER_DIM else 1, dtype=torch.float32, device=dev)
        wm, bm, ls = net.p["act.action_out.fc_mean.weight"], net.p["act.action_out.fc_mean.bias"], net.p["act.action_out.log_std"]
        am, ms = (active, msum) if pol_masks else (None, None)
        _launch("spo_ma_ppo_actor_loss", L.ptr(feat), n, net.H, L.ptr(wm), L.ptr(bm), L.ptr(ls), A, L.ptr(actions), L.ptr(old_logp), L.ptr(adv),
                None, None, L.ptr(factor), L.ptr(am), L.ptr(ms), mode, 1.0 - float(c["clip_param"]), 1.0 + float(c["clip_param"]),
                nets.std_x_coef, nets.std_y_coef, L.ptr(ws["dmean"]), L.ptr(imp), L.ptr(ws["part"]), L.stream())
        scal = torch.empty(3, dtype=torch.float32, device=dev)
        _launch("spo_ma_ppo_actor_finalize", L.ptr(ws["part"]), nb32, n, L.ptr(ms), mode, L.ptr(ls), A, nets.std_x_coef, nets.std_y_coef,
                float(c["entropy_coef"]), L.ptr(net.g["act.action_out.fc_mean.bias"]), L.ptr(net.g["act.action_out.log_std"]), L.ptr(scal),
                L.stream())
        self._vjp_from_mean(net, obs, feat, ws)
        actor_grad_norm = self._clip_adam(net, c["actor_lr"])
        # ---- critic ----
        vm, vs = (active, msum) if val_masks else (None, None)
        value_loss, critic_grad_norm = self._critic_update(nets.critic, share_obs, value_preds, returns, vm, vs)
        self.last_ratio = scal[2]
        return value_loss, critic_grad_norm, scal[0], scal[1], actor_grad_norm, imp

    def train(self, buf, perms=None):
        """mappo.py:165-186 / happo.py:173-194: advantages = returns - denormalised predictions, standardised by the mean and
        unbiased std + 1e-5 over every entry (no NaN masking), then learning_iters whole-batch updates.  ``perms``: the row
        orders to use (one per iteration; torch.randperm on the device when omitted).  Returns the last update's values."""
        advantages = _standardised_advantages(buf.returns, buf.value_preds, *self.popart_mean_sqrt_var())
        out = None
        for it in range(int(self.cfg["learning_iters"])):
            out = self.ppo_update(buf.whole_batch_sample(advantages, None, None if perms is None else perms[it]))
        return out


class MAPPOTrainer(_TwoNetPPOTrainer):
    """``MAPPO_Trainer`` (mappo.py:96-186): each action dimension clipped on its own (imp_weights [n, A]), no cross-agent factor
    in the loss, and the value loss always a plain mean (mappo.py:117 ignores use_value_active_masks)."""
    RATIO_MODE = L.MA_RATIO_PER_DIM
    USES_FACTOR = False
    HONOURS_VALUE_MASKS = False


class HAPPOTrainer(_TwoNetPPOTrainer):
    """``HAPPO_Trainer`` (happo.py:96-194): the product of the per-dimension ratios times the cross-agent factor on the plain
    advantage; both active-mask flags honoured."""
    RATIO_MODE = L.MA_RATIO_PRODUCT
    USES_FACTOR = True
    HONOURS_VALUE_MASKS = True


def _tangent_views(net, buf):
    """Views of a vector in the net's packed layout (buf[P], like net.flat) under the parameter names."""
    base, out = net.flat.data_ptr(), {}
    for k, t in net.p.items():
        off = (t.data_ptr() - base) // t.element_size()
        out[k] = buf[off:off + t.numel()].view(t.shape)
    return out


def macpo_step_coefficients(q, r, s, bb, rescale, target_kl):
    """The scalar part of MACPO_Trainer.trpo_update (macpo.py:264-325) on host values, with the reference's types: q, r, s are
    1-element fp32 tensors, bb (= |b|^2) a 0-dim fp32 tensor, rescale the fp32 constraint value (or the float 1e-8 that replaces
    0).  Returns (optim_case, lam, nu, use_a): the step is x = (xg + nu xb) / (lam + 1e-8) when use_a, else nu xb."""
    import math
    if bb <= 1e-8 and rescale < 0:                     # case 4: no usable cost gradient, constraint satisfied
        r = s = torch.tensor(0)
        pos_cauchy = torch.tensor(0)
        recover = torch.tensor(0)
        optim_case = 4
    else:
        if r == 0:
            r = 1e-8
        if s == 0:
            s = 1e-8
        pos_cauchy = q - (r ** 2) / (1e-8 + s)
        recover = 2 * target_kl - (rescale ** 2) / (1e-8 + s)
        if rescale < 0 and recover < 0:
            optim_case = 3
        elif rescale < 0 and recover >= 0:
            optim_case = 2
        elif rescale >= 0 and recover >= 0:
            optim_case = 1
        else:
            optim_case = 0
    if recover == 0:
        recover = 1e-8
    if optim_case in (3, 4):
        lam = torch.sqrt(q / (2 * target_kl))
        nu = torch.tensor(0)
    elif optim_case in (1, 2):
        LA, LB = [0, r / rescale], [r / rescale, math.inf]
        LA, LB = (LA, LB) if rescale < 0 else (LB, LA)

        def proj(x, L):
            return max(L[0], min(L[1], x))
        lam_a = proj(torch.sqrt(pos_cauchy / recover), LA)
        lam_b = proj(torch.sqrt(q / torch.tensor(2 * target_kl)), LB)

        def f_a(lam):
            return -0.5 * (pos_cauchy / (1e-8 + lam) + recover * lam) - r * rescale / (1e-8 + s)

        def f_b(lam):
            return -0.5 * (q / (1e-8 + lam) + 2 * target_kl * lam)
        lam = lam_a if f_a(lam_a) >= f_b(lam_b) else lam_b
        nu = max(0, lam * rescale - r) / (1e-8 + s)
    else:
        lam = torch.tensor(0)
        nu = torch.sqrt(torch.tensor(2 * target_kl) / (1e-8 + s))
    return optim_case, lam, nu, optim_case > 0


class MACPOTrainer(_AgentTrainer):
    """``MACPO_Trainer`` (safepo/multi_agent/macpo.py:96-415) for one agent around ``MultiAgentNets``.  The critics are updated
    exactly as in MAPPO-Lag (the shared ``_critic_update``); the actor takes one constrained trust-region step: the gradients g / b of the
    reward / cost ratio surrogates (spo_ma_ratio_loss + the backward chain), two conjugate-gradient solves against F + 0.1 I
    (Fisher-vector products from spo_ma_mlp_layer_jvp / spo_ma_head_jvp, the backward chain and spo_ma_fvp_finalize), the case
    analysis on host values after one read of q, r, s, |b|^2, and a backtracking line search that reads 8 floats per trial
    (reward loss, cost loss, KL, mean ratio, -x.g, |x|^2).
    ``cfg`` adds the reference's target_kl, searching_steps, step_fraction, fraction_coef and conjugate_gradient_iters."""

    CG_DAMPING = 0.1            # macpo.py:198
    CG_RESIDUAL_TOL = 1e-10     # macpo.py:169

    def __init__(self, nets: MultiAgentNets, cfg):
        super().__init__(nets, cfg)
        net, dev = nets.actor, self.device
        P = net.flat.numel()
        f = dict(dtype=torch.float32, device=dev)
        self.P = P
        self.old_flat = torch.zeros(P, **f)          # the old actor (macpo.py:329-335) as a copy of the packed buffer
        self._v = {k: torch.zeros(P, **f) for k in ("g", "b", "xg", "xb", "x", "r", "p", "Ap")}
        self._work = torch.zeros(L.lib().spo_ma_work_floats(), **f)
        self._cg_state = torch.zeros(4, **f)
        self._scal = torch.zeros(4 + 2 * 32, **f)   # q, r, s, |b|^2, reward surrogate [A], cost surrogate [A]
        self._ls = torch.zeros(8, **f)              # trial: reward loss, cost loss, KL, mean ratio, -x.g, |x|^2
        self._ls_off = (net.p["act.action_out.log_std"].data_ptr() - net.flat.data_ptr()) // 4
        self._tan = {}
        self.last = {}

    def _tangent_bufs(self, n, H):
        if (n, H) not in self._tan:
            self._tan[(n, H)] = (torch.empty(n, H, dtype=torch.float32, device=self.device),
                                 torch.empty(n, H, dtype=torch.float32, device=self.device))
        return self._tan[(n, H)]

    # ---- pieces ----
    def actor_forward(self, obs):
        """Training forward of the actor at its current weights (activations kept for fvp) and the means [n, A]."""
        net, n, A = self.nets.actor, obs.shape[0], self.nets.act_dim
        ws = self._ws(n, net)
        feat = self._forward_train(net, obs, ws)
        mean = self.nets.head(net, feat, ws.setdefault("mean_old", torch.empty(n, A, dtype=torch.float32, device=self.device)))
        self._obs, self._feat, self._fws = obs, feat, ws
        return mean

    def fvp(self, v, out):
        """out = (F + 0.1 I) v for the actor at the weights of the last actor_forward (macpo.py:187-198): F is the Hessian of
        mean_rows(sum_j KL_j) at new = old.  v, out: [P] in the packed layout."""
        nets, net, ws, obs, feat = self.nets, self.nets.actor, self._fws, self._obs, self._feat
        p, n, H, A = net.p, obs.shape[0], net.H, nets.act_dim
        tv = _tangent_views(net, v)
        a, b = self._tangent_bufs(n, H)
        w, bb, lw, lb = net.blocks[0]
        fw, fb = "base.feature_norm.weight", "base.feature_norm.bias"
        _launch("spo_ma_mlp_layer_jvp", L.ptr(obs), None, n, net.D, L.ptr(p[w]), L.ptr(tv[w]), L.ptr(tv[bb]), L.ptr(ws["pre"][0]), L.ptr(p[lw]),
                L.ptr(tv[lw]), L.ptr(tv[lb]), H, L.ptr(p[fw]), L.ptr(p[fb]), L.ptr(tv[fw]), L.ptr(tv[fb]), L.ptr(a), L.stream())
        for i, (w, bb, lw, lb) in enumerate(net.blocks[1:], start=1):
            _launch("spo_ma_mlp_layer_jvp", L.ptr(ws["out"][i - 1]), L.ptr(a), n, H, L.ptr(p[w]), L.ptr(tv[w]), L.ptr(tv[bb]), L.ptr(ws["pre"][i]),
                    L.ptr(p[lw]), L.ptr(tv[lw]), L.ptr(tv[lb]), H, None, None, None, None, L.ptr(b), L.stream())
            a, b = b, a
        wm, bm, ls = "act.action_out.fc_mean.weight", "act.action_out.fc_mean.bias", "act.action_out.log_std"
        _launch("spo_ma_head_jvp", L.ptr(feat), L.ptr(a), n, H, L.ptr(p[wm]), L.ptr(tv[wm]), L.ptr(tv[bm]), A, L.ptr(p[ls]), nets.std_x_coef,
                nets.std_y_coef, L.ptr(ws["dmean"]), L.ptr(ws["part"]), L.stream())
        _launch("spo_ma_partial_reduce", L.ptr(ws["part"]), (n + 31) // 32, A, 1, A, L.ptr(net.g[bm]), None, None, 1.0, L.stream())
        self._vjp_from_mean(net, obs, feat, ws)
        _launch("spo_ma_fvp_finalize", L.ptr(net.gflat), L.ptr(v), L.ptr(out), self.P, L.ptr(p[ls]), self._ls_off, A, nets.std_x_coef,
                nets.std_y_coef, self.CG_DAMPING, L.stream())
        return out

    def surrogate_grad(self, mean, actions, old_logp, adv, factor, sign, loss_out, grad_out):
        """grad_out[P] = d/d params of sign * mean(ratio * factor * adv) (macpo.py:239-251); loss_out[0] = that loss."""
        nets, net, ws, obs, feat = self.nets, self.nets.actor, self._fws, self._obs, self._feat
        n, A = obs.shape[0], nets.act_dim
        ls = net.p["act.action_out.log_std"]
        _launch("spo_ma_ratio_loss", L.ptr(mean), n, L.ptr(ls), A, L.ptr(actions), L.ptr(old_logp), L.ptr(adv), L.ptr(factor), float(sign),
                nets.std_x_coef, nets.std_y_coef, L.ptr(ws["dmean"]), L.ptr(ws["part"]), L.stream())
        nb32 = (n + 31) // 32
        _launch("spo_ma_partial_reduce", L.ptr(ws["part"]), nb32, 3 * A, 1, A, L.ptr(loss_out), None, None, float(sign) / n, L.stream())
        _launch("spo_ma_partial_reduce", L.ptr(ws["part"]), nb32, 3 * A, 3, A, None, L.ptr(net.g["act.action_out.fc_mean.bias"]),
                L.ptr(net.g["act.action_out.log_std"]), 1.0, L.stream())
        self._vjp_from_mean(net, obs, feat, ws)
        grad_out.copy_(net.gflat)
        return grad_out

    def conjugate_gradient(self, b, x):
        """MACPO's CG (macpo.py:168-185) for (F + 0.1 I) x = b, conjugate_gradient_iters steps, no host synchronisation (the
        residual break is a device flag)."""
        v, P, st = self._v, self.P, self._cg_state
        _launch("spo_ma_cg_begin", L.ptr(b), L.ptr(x), L.ptr(v["r"]), L.ptr(v["p"]), P, L.ptr(self._work), L.ptr(st), L.stream())
        for _ in range(int(self.cfg["conjugate_gradient_iters"])):
            self.fvp(v["p"], v["Ap"])
            _launch("spo_ma_dots", L.ptr(v["p"]), L.ptr(v["Ap"]), None, None, None, None, None, None, 1, P, L.ptr(self._work), L.ptr(st[1:]), L.stream())
            _launch("spo_ma_cg_update", L.ptr(x), L.ptr(v["r"]), L.ptr(v["p"]), L.ptr(v["Ap"]), P, self.CG_RESIDUAL_TOL, L.ptr(self._work),
                    L.ptr(st), L.stream())
        return x

    def linesearch_eval(self, obs, mean_old, actions, old_logp, adv, cost_adv, factor, out):
        """out[0:4] = (reward loss, cost loss, mean KL(old || new), mean ratio) of the actor's current weights against the old
        actor (macpo.py:349-368)."""
        nets, net, n, A = self.nets, self.nets.actor, obs.shape[0], self.nets.act_dim
        feat = net.features(obs, nets._buffers(n, net.H))
        ws = self._fws
        mean = nets.head(net, feat, ws.setdefault("mean_new", torch.empty(n, A, dtype=torch.float32, device=self.device)))
        p = net.p
        old_ls = self.old_flat[self._ls_off:self._ls_off + A]
        _launch("spo_ma_linesearch_eval", L.ptr(mean), L.ptr(mean_old), L.ptr(p["act.action_out.log_std"]), L.ptr(old_ls), A, L.ptr(actions),
                L.ptr(old_logp), L.ptr(adv), L.ptr(cost_adv), L.ptr(factor), n, nets.std_x_coef, nets.std_y_coef, L.ptr(self._work), L.ptr(out),
                L.stream())
        return out

    # ---- the update ----
    def trpo_update(self, sample):
        """One MACPO_Trainer.trpo_update (macpo.py:200-380) on the whole sample.  Returns a dict of the logged quantities
        (value_loss, critic_grad_norm, cost_loss = the actor's cost surrogate -- which the reference logs as the cost critic's
        loss --, cost_critic_loss, cost_grad_norm, kl, loss_improve, expected_improve, dist_entropy, ratio = mean importance
        ratio of the last trial) and of the step (q, r, s, optim_case, lam, nu, accepted = index of the accepted trial or -1)."""
        c, nets, net = self.cfg, self.nets, self.nets.actor
        (obs, share_obs, actions, old_logp, value_preds, returns, adv, factor, _, cost_preds, cost_returns, cost_adv,
         aver_costs) = self._device_sample(sample)
        n, A = obs.shape[0], nets.act_dim
        # ---- critics, as MAPPO-Lag (macpo.py:215-231) ----
        value_loss, critic_grad_norm = self._critic_update(nets.critic, share_obs, value_preds, returns)
        cost_critic_loss, cost_grad_norm = self._critic_update(nets.cost_critic, share_obs, cost_preds, cost_returns)
        # ---- constraint value (macpo.py:234-237): fp32, like the reference's tensor ----
        rescale = (torch.as_tensor(aver_costs, dtype=torch.float32).mean().cpu() - float(c["cost_limit"])) * (1 - float(c["gamma"]))
        if rescale == 0:
            rescale = 1e-8
        # ---- surrogate gradients, CG solves, q / r / s ----
        mean_old = self.actor_forward(obs)
        self.old_flat.copy_(net.flat)
        v, sc, P = self._v, self._scal, self.P
        self.surrogate_grad(mean_old, actions, old_logp, adv, factor, -1.0, sc[4:4 + A], v["g"])
        self.surrogate_grad(mean_old, actions, old_logp, cost_adv, factor, 1.0, sc[36:36 + A], v["b"])
        self.conjugate_gradient(v["g"], v["xg"])
        self.conjugate_gradient(v["b"], v["xb"])
        _launch("spo_ma_dots", L.ptr(v["g"]), L.ptr(v["xg"]), L.ptr(v["g"]), L.ptr(v["xb"]), L.ptr(v["b"]), L.ptr(v["xb"]), L.ptr(v["b"]), L.ptr(v["b"]),
                4, P, L.ptr(self._work), L.ptr(sc), L.stream())
        host = sc.cpu()                                   # the one read before the case analysis
        q, r, s, bb = host[0:1].clone(), host[1:2].clone(), host[2:3].clone(), host[3].clone()
        reward_loss, cost_loss = host[4].clone(), host[36].clone()
        target_kl = float(c["target_kl"])
        optim_case, lam, nu, use_a = macpo_step_coefficients(q, r, s, bb, rescale, target_kl)
        coef = (1.0 / (lam + 1e-8)) if use_a else 0.0
        _launch("spo_ma_step_dir", L.ptr(v["xg"]), L.ptr(v["xb"]), float(coef), float(nu), int(use_a), L.ptr(v["x"]), P, L.stream())
        ls = self._ls
        _launch("spo_ma_dots", L.ptr(v["x"]), L.ptr(v["g"]), None, None, None, None, None, None, 1, P, L.ptr(self._work), L.ptr(ls[4:]), L.stream())
        # ---- line search (macpo.py:337-378) ----
        fraction, fraction_coef = float(c["step_fraction"]), float(c["fraction_coef"])
        accepted, expected_improve, out = -1, None, None
        ls_param = net.p["act.action_out.log_std"]
        for i in range(int(c["searching_steps"])):
            _launch("spo_ma_dots", L.ptr(v["x"]), L.ptr(v["x"]), None, None, None, None, None, None, 1, P, L.ptr(self._work), L.ptr(ls[5:]), L.stream())
            _launch("spo_ma_ls_trial", L.ptr(self.old_flat), L.ptr(v["x"]), L.ptr(ls[5:]), float(fraction_coef * (fraction ** i)), L.ptr(net.flat), P,
                    L.stream())
            self.linesearch_eval(obs, mean_old, actions, old_logp, adv, cost_adv, factor, ls)
            out = ls.cpu()
            if expected_improve is None:
                expected_improve = -out[4:5].clone()
            new_reward_loss, new_cost_loss, kl = out[0].clone(), out[1].clone(), out[2].clone()
            loss_improve = new_reward_loss - reward_loss
            if (kl < target_kl) and (loss_improve < 0 if optim_case > 1 else True) and (new_cost_loss - cost_loss <= max(-rescale, 0)):
                accepted = i
                break
            expected_improve *= fraction
        std = torch.sigmoid(ls_param / nets.std_x_coef) * nets.std_y_coef       # the last trial's entropy (act.py:57-60)
        dist_entropy = (0.5 + _LOG_SQRT_2PI + std.log()).mean()
        if accepted < 0:
            net.flat.copy_(self.old_flat)
        self.last = dict(value_loss=value_loss, critic_grad_norm=critic_grad_norm, cost_loss=cost_loss, cost_critic_loss=cost_critic_loss,
                         cost_grad_norm=cost_grad_norm, kl=kl, loss_improve=loss_improve, expected_improve=expected_improve,
                         dist_entropy=dist_entropy, ratio=out[3].clone(), q=q, r=r, s=s, bb=bb, rescale=rescale, reward_loss=reward_loss,
                         optim_case=optim_case, lam=lam, nu=nu, accepted=accepted)
        return self.last

    def train(self, buf, perms=None):
        """MACPO_Trainer.train (macpo.py:382-400): advantages standardised with std + 1e-5 over all entries (no NaN masking),
        then ONE trpo_update on the whole batch (num_mini_batch = 1).  ``perms``: [row order] (torch.randperm on the device
        when omitted)."""
        mean, sd = self.popart_mean_sqrt_var()
        advantages = _standardised_advantages(buf.returns, buf.value_preds, mean, sd)
        cost_adv = _standardised_advantages(buf.cost_returns, buf.cost_preds, mean, sd)
        return self.trpo_update(buf.whole_batch_sample(advantages, cost_adv, None if perms is None else perms[0]))
