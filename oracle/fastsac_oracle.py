"""CPU oracle for the FastSAC update — TEST INFRASTRUCTURE, NOT PRODUCT CODE (same rules as oracle/ppo_oracle.py).

Restates rl_x/algorithms/fastsac/pytorch/{policy,q_network,critic,entropy_coefficient,observation_normalizer,fastsac}.py
(nico-bohlinger/RL-X @ 46d8e26), fp32 path (bf16 autocast off), in plain PyTorch with autograd:
  * policy torso Linear-LayerNorm-SiLU x3 (512, 256, 128), mean / log_std heads, tanh log-std squash (policy.py:36-62), tanh-Gaussian
    action with the action_scale log-prob correction (policy.py:64-75);
  * Q network Linear-LayerNorm-SiLU x3 (768, 384, 192) -> nr_atoms logits on [state | action] (q_network.py:20-38);
  * C51 target: entropy-adjusted n-step return, clamp to [v_min, v_max], projection with the integer-bin fix-up, cross-entropy
    (fastsac.py:143-205); entropy-coefficient loss (:228-236); polyak (:316-320); policy loss on the expected Q (:106-124);
  * observation normaliser running statistics (observation_normalizer.py:28-47);
  * torch.optim.AdamW(lr, weight_decay, betas) for the three optimisers (fastsac.py:87-89) — the same torch primitive the reference calls.
The normal draws of Normal.rsample() are inputs.

Parity status: PINNED against `tests/golden/fastsac_update.npz`, captured from the executed reference by
`tests/golden/make_golden_fastsac.py` (checked by tests/test_oracle_vs_reference.py::test_fastsac_update_matches_reference).
"""
import math

import torch
import torch.nn.functional as F

POLICY_WIDTHS = (512, 256, 128)
Q_WIDTHS = (768, 384, 192)


def reference_init(obs, act, nr_atoms, seed):
    """The parameter values FastSAC.__init__ produces (fastsac.py:77-84): same torch modules, same construction order, same seed."""
    torch.manual_seed(seed)

    def torso(inp, widths):
        layers, last = [], inp
        for w in widths:
            layers += [torch.nn.Linear(last, w), torch.nn.LayerNorm(w)]
            last = w
        return layers

    pol_layers = torso(obs, POLICY_WIDTHS)
    mean, log_std = torch.nn.Linear(128, act), torch.nn.Linear(128, act)
    for lyr in (mean, log_std):
        torch.nn.init.constant_(lyr.weight, 0.0)
        torch.nn.init.constant_(lyr.bias, 0.0)
    pol = {"torso": [(l.weight.detach().clone(), l.bias.detach().clone()) for l in pol_layers],
           "mean": (mean.weight.detach().clone(), mean.bias.detach().clone()), "log_std": (log_std.weight.detach().clone(), log_std.bias.detach().clone())}

    def qnet():
        layers = torso(obs + act, Q_WIDTHS)
        head = torch.nn.Linear(192, nr_atoms)
        return {"torso": [(l.weight.detach().clone(), l.bias.detach().clone()) for l in layers], "head": (head.weight.detach().clone(), head.bias.detach().clone())}

    q1, q2 = qnet(), qnet()
    qnet(), qnet()  # the two target networks consume the generator too before being overwritten (critic.py:16-19)
    return pol, q1, q2


def _leaves(net):
    out = []
    for w, b in net["torso"]:
        out += [w, b]
    for k in ("mean", "log_std", "head"):
        if k in net:
            out += list(net[k])
    return out


def _clone(net, grad, dtype=torch.float32):
    f = (lambda t: t.detach().to(dtype, copy=True).requires_grad_(True)) if grad else (lambda t: t.detach().to(dtype, copy=True))
    out = {"torso": [(f(w), f(b)) for w, b in net["torso"]]}
    for k in ("mean", "log_std", "head"):
        if k in net:
            out[k] = (f(net[k][0]), f(net[k][1]))
    return out


def torso_forward(net, x):
    """Linear -> LayerNorm(eps 1e-5) -> SiLU per block; net["torso"] alternates (Linear w, b), (LayerNorm w, b)."""
    t = net["torso"]
    for i in range(0, len(t), 2):
        x = F.linear(x, t[i][0], t[i][1])
        x = F.layer_norm(x, (x.shape[-1],), t[i + 1][0], t[i + 1][1], eps=1e-5)
        x = F.silu(x)
    return x


def policy_forward(pol, x, log_std_min, log_std_max):
    latent = torso_forward(pol, x)
    mean = F.linear(latent, *pol["mean"])
    log_std = torch.tanh(F.linear(latent, *pol["log_std"]))
    return mean, log_std_min + 0.5 * (log_std_max - log_std_min) * (log_std + 1)


def action_and_log_prob(pol, x, eps, action_scale, log_std_min, log_std_max):
    """policy.py:64-75 with rsample() = mean + std * eps."""
    mean, log_std = policy_forward(pol, x, log_std_min, log_std_max)
    std = log_std.exp()
    raw = mean + std * eps
    th = torch.tanh(raw)
    log_prob = -((raw - mean) ** 2) / (2 * std ** 2) - log_std - math.log(math.sqrt(2 * math.pi))
    log_prob = log_prob - torch.log((1 - th.pow(2)) + 1e-6) - torch.log(action_scale + 1e-6)
    return th * action_scale, log_prob.sum(1)


def q_forward(q, x, a):
    return F.linear(torso_forward(q, torch.cat([x, a], dim=1)), *q["head"])


class Normalizer:
    """observation_normalizer.py:10-47."""

    def __init__(self, obs, eps=1e-8):
        self.mean, self.var, self.std, self.count, self.eps = torch.zeros(1, obs), torch.ones(1, obs), torch.ones(1, obs), 0, eps

    def update(self, x):
        bm, bv, bc = x.mean(0, keepdim=True), x.var(0, unbiased=False, keepdim=True), x.shape[0]
        new_count = self.count + bc
        delta = bm - self.mean
        self.mean = self.mean + delta * bc / new_count
        delta2 = bm - self.mean
        m2 = self.var * self.count + bv * bc + delta2.pow(2) * self.count * bc / new_count
        self.var = m2 / new_count
        self.std = self.var.sqrt()
        self.count = new_count

    def normalize(self, x, update):
        if update:
            self.update(x)
        return (x - self.mean) / (self.std + self.eps)


class Learner:
    def __init__(self, pol, q1, q2, action_scale, lr, weight_decay, betas, gamma, tau, v_min, v_max, nr_atoms, target_entropy, alpha_init,
                 log_std_min, log_std_max, clipped_double_q=False, max_grad_norm=-1.0, dtype=torch.float32):
        """dtype: the precision of every tensor of the learner (float32: the reference's; float64: the yardstick of the GPU tests, which pass
        a float64 action_scale and float64 batches).  The tensors stay on the device of `pol`."""
        self.clipped, self.max_grad_norm = clipped_double_q, max_grad_norm
        self.pol, self.q1, self.q2 = _clone(pol, True, dtype), _clone(q1, True, dtype), _clone(q2, True, dtype)
        self.q1t, self.q2t = _clone(q1, False, dtype), _clone(q2, False, dtype)
        dev = self.pol["mean"][0].device
        self.log_alpha = torch.full((1,), math.log(alpha_init), dtype=dtype, device=dev, requires_grad=True)
        self.popt = torch.optim.AdamW(_leaves(self.pol), lr=lr, weight_decay=weight_decay, betas=betas)
        self.qopt = torch.optim.AdamW(_leaves(self.q1) + _leaves(self.q2), lr=lr, weight_decay=weight_decay, betas=betas)
        self.aopt = torch.optim.AdamW([self.log_alpha], lr=lr, weight_decay=weight_decay, betas=betas)
        self.action_scale, self.gamma, self.tau, self.v_min, self.v_max, self.nr_atoms = action_scale, gamma, tau, v_min, v_max, nr_atoms
        self.target_entropy, self.lsmin, self.lsmax = target_entropy, log_std_min, log_std_max
        self.support = torch.linspace(v_min, v_max, nr_atoms, dtype=dtype, device=dev)

    def critic_and_entropy_step(self, s, ns, a, r, dones, truncs, eff, eps_next):
        """fastsac.py:141-238, then the polyak update of :316-320."""
        with torch.no_grad():
            na, nlp = action_and_log_prob(self.pol, ns, eps_next, self.action_scale, self.lsmin, self.lsmax)
            delta_z = (self.v_max - self.v_min) / (self.nr_atoms - 1)
            bootstrap = 1.0 - (dones * (1.0 - truncs))
            discount = (self.gamma ** eff) * bootstrap
            adj_r = r - discount * self.log_alpha.exp() * nlp
            target_z = torch.clamp(adj_r.unsqueeze(1) + discount.unsqueeze(1) * self.support.unsqueeze(0), self.v_min, self.v_max)
            b = (target_z - self.v_min) / delta_z
            lo0, up0 = torch.floor(b).long(), torch.ceil(b).long()
            is_int = lo0 == up0                                   # b on a bin: move one neighbour so that the two weights still sum to 1
            lo = torch.where(is_int & (lo0 > 0), lo0 - 1, lo0)
            up = torch.where(is_int & (lo0 == 0), up0 + 1, up0)
            d1 = F.softmax(q_forward(self.q1t, ns, na), dim=1)
            d2 = F.softmax(q_forward(self.q2t, ns, na), dim=1)
            wl, wu = up.to(b.dtype) - b, b - lo.to(b.dtype)
            proj1, proj2 = torch.zeros_like(d1), torch.zeros_like(d2)
            for proj, d in ((proj1, d1), (proj2, d2)):
                proj.scatter_add_(1, lo, d * wl)
                proj.scatter_add_(1, up, d * wu)
            q1_next_value = (proj1 * self.support).sum(1)
            if self.clipped:  # fastsac.py:179-182: both critics learn the distribution of the smaller next value
                q2_next_value = (proj2 * self.support).sum(1)
                proj1 = proj2 = torch.where(q1_next_value.unsqueeze(1) < q2_next_value.unsqueeze(1), proj1, proj2)
        l1 = -(proj1 * F.log_softmax(q_forward(self.q1, s, a), dim=1)).sum(1).mean()
        l2 = -(proj2 * F.log_softmax(q_forward(self.q2, s, a), dim=1)).sum(1).mean()
        q_loss = l1 + l2
        self.qopt.zero_grad()
        q_loss.backward()
        if self.max_grad_norm != -1.0:   # fastsac.py:203-210
            cg = float(torch.nn.utils.clip_grad_norm_(_leaves(self.q1) + _leaves(self.q2), self.max_grad_norm))
        else:
            cg = math.sqrt(sum(float(p.grad.norm(2) ** 2) for p in _leaves(self.q1) + _leaves(self.q2)))
        self.qopt.step()
        entropy = -nlp
        ent_loss = (self.log_alpha.exp() * (entropy - self.target_entropy)).mean()
        self.aopt.zero_grad()
        ent_loss.backward()
        eg = float(self.log_alpha.grad.norm(2) ** 2)
        self.aopt.step()
        with torch.no_grad():
            for tgt, src in ((self.q1t, self.q1), (self.q2t, self.q2)):
                for pt, ps in zip(_leaves(tgt), _leaves(src)):
                    pt.mul_(1.0 - self.tau).add_(ps.detach(), alpha=self.tau)
        return {"loss/q_loss": q_loss.item(), "loss/entropy_loss": ent_loss.item(), "q/q_min": q1_next_value.min().item(),
                "q/q_max": q1_next_value.max().item(), "entropy/entropy": entropy.mean().item(), "gradients/critic_grad_norm": cg,
                "gradients/entropy_grad_norm": eg}

    def policy_step(self, s, eps):
        """fastsac.py:106-138."""
        a, lp = action_and_log_prob(self.pol, s, eps, self.action_scale, self.lsmin, self.lsmax)
        v1 = (F.softmax(q_forward(self.q1, s, a), dim=1) * self.support).sum(1)
        v2 = (F.softmax(q_forward(self.q2, s, a), dim=1) * self.support).sum(1)
        qv = torch.minimum(v1, v2) if self.clipped else (v1 + v2) / 2.0   # fastsac.py:117-120
        alpha = self.log_alpha.exp().detach()
        loss = (alpha * lp - qv).mean()
        self.popt.zero_grad()
        for p in _leaves(self.q1) + _leaves(self.q2):
            p.grad = None
        loss.backward()
        if self.max_grad_norm != -1.0:   # fastsac.py:126-133
            pg = float(torch.nn.utils.clip_grad_norm_(_leaves(self.pol), self.max_grad_norm))
        else:
            pg = math.sqrt(sum(float(p.grad.norm(2) ** 2) for p in _leaves(self.pol)))
        self.popt.step()
        return {"loss/policy_loss": loss.item(), "entropy/alpha": alpha.item(), "gradients/policy_grad_norm": pg}
