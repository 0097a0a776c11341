"""CPU oracle for the SAC update path — TEST INFRASTRUCTURE, NOT PRODUCT CODE (same rules as oracle/ppo_oracle.py).

Plain-PyTorch (CPU, fp32, autograd) restatement of rl_x/algorithms/sac/pytorch/{policy,q_network,critic,entropy_coefficient,sac}.py
(nico-bohlinger/RL-X @ 46d8e26); each function cites the lines it follows.  Parity status: PINNED against vectors captured from the
executed reference (`tests/golden/make_golden_sac.py` -> `tests/golden/sac_small.npz`, checked by tests/test_oracle_vs_reference.py):
six consecutive updates from the reference's initial weights, sampled batches and rsample noise reproduce its final weights,
temperature and every logged loss / gradient norm.
"""
import math

import torch
import torch.nn.functional as F

POLICY_KEYS = ["torso.0.weight", "torso.0.bias", "torso.2.weight", "torso.2.bias", "mean.weight", "mean.bias", "log_std.weight", "log_std.bias"]
Q_KEYS = ["critic.0.weight", "critic.0.bias", "critic.2.weight", "critic.2.bias", "critic.4.weight", "critic.4.bias"]


def init_params(obs, act, hidden, seed=0):
    """Default nn.Linear initialisation as the reference modules use it (policy.py:34-43, q_network.py:27-33)."""
    torch.manual_seed(seed)
    import torch.nn as nn
    pol = {}
    for name, lin in [("torso.0", nn.Linear(obs, hidden)), ("torso.2", nn.Linear(hidden, hidden)), ("mean", nn.Linear(hidden, act)),
                      ("log_std", nn.Linear(hidden, act))]:
        pol[name + ".weight"], pol[name + ".bias"] = lin.weight.detach().clone(), lin.bias.detach().clone()

    def qnet():
        d = {}
        for i, lin in zip((0, 2, 4), (nn.Linear(obs + act, hidden), nn.Linear(hidden, hidden), nn.Linear(hidden, 1))):
            d[f"critic.{i}.weight"], d[f"critic.{i}.bias"] = lin.weight.detach().clone(), lin.bias.detach().clone()
        return d
    return pol, qnet(), qnet()


def policy_get_action(pol, x, eps, low, high, ls_min=-20.0, ls_max=2.0):
    """ref: policy.py:45-64 with normal.rsample() == mean + std * eps."""
    h = F.relu(F.linear(x, pol["torso.0.weight"], pol["torso.0.bias"]))
    h = F.relu(F.linear(h, pol["torso.2.weight"], pol["torso.2.bias"]))
    mean = F.linear(h, pol["mean.weight"], pol["mean.bias"])
    log_std = torch.clamp(F.linear(h, pol["log_std.weight"], pol["log_std.bias"]), ls_min, ls_max)
    std = torch.exp(log_std)
    normal = torch.distributions.Normal(mean, std)
    action = mean + std * eps
    action_tanh = torch.tanh(action)
    log_prob = normal.log_prob(action)
    log_prob = log_prob - torch.log((1 - action_tanh.pow(2)) + 1e-6)
    log_prob = log_prob.sum(1, keepdim=True)
    scaled = low + (0.5 * (action_tanh + 1.0) * (high - low))
    return action_tanh, scaled, log_prob


def policy_deterministic(pol, x, low, high):
    """ref: policy.py:67-73."""
    h = F.relu(F.linear(x, pol["torso.0.weight"], pol["torso.0.bias"]))
    h = F.relu(F.linear(h, pol["torso.2.weight"], pol["torso.2.bias"]))
    return low + (0.5 * (torch.tanh(F.linear(h, pol["mean.weight"], pol["mean.bias"])) + 1.0) * (high - low))


def q_forward(q, x, a):
    """ref: q_network.py:36-38."""
    h = torch.cat([x, a], dim=1)
    h = F.relu(F.linear(h, q["critic.0.weight"], q["critic.0.bias"]))
    h = F.relu(F.linear(h, q["critic.2.weight"], q["critic.2.bias"]))
    return F.linear(h, q["critic.4.weight"], q["critic.4.bias"])


class Learner:
    """ref: SAC.__init__ optimisers (sac.py:74-77) and one iteration of the optimisation block (sac.py:219-259)."""

    def __init__(self, pol, q1, q2, low, high, lr=3e-4, gamma=0.99, tau=0.005, target_entropy=None, ls_min=-20.0, ls_max=2.0, log_alpha=0.0,
                 q1_target=None, q2_target=None, dtype=torch.float32, device="cpu"):
        """dtype / device: where the learner's parameters, log_alpha and action bounds live (the caller's batches must match).  The float32
        CPU default is the pinned oracle; float64 is the high-precision reference of the GPU tests."""
        to = lambda v: v.to(device, dtype).clone()
        g = lambda d: {k: to(v).requires_grad_(True) for k, v in d.items()}
        self.pol, self.q1, self.q2 = g(pol), g(q1), g(q2)
        self.q1t = {k: to(v) for k, v in (q1_target or q1).items()}
        self.q2t = {k: to(v) for k, v in (q2_target or q2).items()}
        self.log_alpha = torch.full((1,), float(log_alpha), dtype=dtype, device=device, requires_grad=True)
        low, high = low.to(device, dtype), high.to(device, dtype)
        self.popt = torch.optim.Adam([self.pol[k] for k in POLICY_KEYS], lr=lr)
        self.qopt = torch.optim.Adam([self.q1[k] for k in Q_KEYS] + [self.q2[k] for k in Q_KEYS], lr=lr)
        self.aopt = torch.optim.Adam([self.log_alpha], lr=lr)
        self.low, self.high, self.gamma, self.tau, self.ls_min, self.ls_max = low, high, gamma, tau, ls_min, ls_max
        self.target_entropy = target_entropy if target_entropy is not None else -float(low.numel())

    def update(self, states, next_states, actions, rewards, dones, eps_next, eps_cur):
        # critic_loss_fn, sac.py:129-159
        with torch.no_grad():
            na, _, nlp = policy_get_action(self.pol, next_states, eps_next, self.low, self.high, self.ls_min, self.ls_max)
            mq = torch.minimum(q_forward(self.q1t, next_states, na), q_forward(self.q2t, next_states, na))
            alpha = self.log_alpha.exp().detach()
            y = rewards.reshape(-1, 1) + self.gamma * (1 - dones.reshape(-1, 1)) * (mq - alpha * nlp)
        q1, q2 = q_forward(self.q1, states, actions), q_forward(self.q2, states, actions)
        q_loss = (F.mse_loss(q1, y) + F.mse_loss(q2, y)) / 2
        self.qopt.zero_grad()
        q_loss.backward()
        # the critic gradient of this update: policy_loss.backward() below accumulates into the same .grad tensors
        self.q_grads = ({k: self.q1[k].grad.clone() for k in Q_KEYS}, {k: self.q2[k].grad.clone() for k in Q_KEYS})
        n1 = math.sqrt(sum(float(self.q1[k].grad.norm(2) ** 2) for k in Q_KEYS))
        n2 = math.sqrt(sum(float(self.q2[k].grad.norm(2) ** 2) for k in Q_KEYS))
        self.qopt.step()
        # Polyak, sac.py:238-242
        with torch.no_grad():
            for src, dst in ((self.q1, self.q1t), (self.q2, self.q2t)):
                for k in Q_KEYS:
                    dst[k].mul_(1.0 - self.tau).add_(src[k].data, alpha=self.tau)
        # policy_and_entropy_loss_fn, sac.py:91-126
        a, _, lp = policy_get_action(self.pol, states, eps_cur, self.low, self.high, self.ls_min, self.ls_max)
        min_q = torch.minimum(q_forward(self.q1, states, a), q_forward(self.q2, states, a))
        alpha = self.log_alpha.exp()
        policy_loss = (alpha.detach() * lp - min_q).mean()
        self.popt.zero_grad()
        policy_loss.backward()
        pn = math.sqrt(sum(float(self.pol[k].grad.norm(2) ** 2) for k in POLICY_KEYS))
        self.popt.step()
        entropy = -lp.detach()
        entropy_loss = (self.log_alpha.exp() * (entropy - self.target_entropy)).mean()
        self.aopt.zero_grad()
        entropy_loss.backward()
        en = float(self.log_alpha.grad.norm(2) ** 2)
        self.aopt.step()
        return {"entropy/alpha": float(alpha), "entropy/entropy": float(entropy.mean()), "gradients/policy_grad_norm": pn,
                "gradients/critic_grad_norm": n1 + n2, "gradients/entropy_grad_norm": en, "loss/q_loss": float(q_loss),
                "loss/policy_loss": float(policy_loss), "loss/entropy_loss": float(entropy_loss), "q_value/q_value": float(min_q.mean())}
