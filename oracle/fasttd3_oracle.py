"""CPU oracle for the FastTD3 update — TEST INFRASTRUCTURE, NOT PRODUCT CODE (same rules as oracle/ppo_oracle.py).

Restates rl_x/algorithms/fasttd3/pytorch/{policy,q_network,critic,fasttd3}.py (nico-bohlinger/RL-X), fp32 path (bf16 autocast off), in
plain PyTorch with autograd:
  * policy Linear-ReLU x3 (512, 256, 128) -> Linear(act) -> tanh, last layer normal_(0, 0.01) / zero bias (policy.py:33-48); acting adds
    noise * per-env scale and optionally clips and rescales to the action bounds (policy.py:57-66);
  * Q network Linear-ReLU x3 (1024, 512, 256) -> nr_atoms logits on [state | action] (q_network.py:27-40);
  * critic target: online policy on s' plus clamped smoothing noise, n-step return, C51 projection with the integer-bin fix-up,
    clipped double-Q selection, cross-entropy (fasttd3.py:139-205); polyak (:316-320); actor loss -mean(min / mean of E[q]) (:104-120);
  * torch.optim.AdamW(lr, weight_decay) for the two optimisers (fasttd3.py:88-89) — the same torch primitive the reference calls.
The normal draws of torch.randn_like are inputs.  The observation normaliser is FastSAC's (oracle/fastsac_oracle.py: byte-identical module).

Parity status: PINNED against `tests/golden/fasttd3_update*.npz`, captured from the executed reference by
`tests/golden/make_golden_fasttd3.py` (checked by tests/test_fasttd3_emulation.py::test_oracle_reproduces_the_reference_run).
"""
import math

import torch
import torch.nn.functional as F

from oracle.fastsac_oracle import Normalizer  # noqa: F401  (re-exported: observation_normalizer.py is the same file in both)

POLICY_WIDTHS = (512, 256, 128)
Q_WIDTHS = (1024, 512, 256)


def _mlp(inp, widths, out):
    layers, last = [], inp
    for w in tuple(widths) + (out,):
        layers.append(torch.nn.Linear(last, w))
        last = w
    return layers


def reference_init(obs, act, nr_atoms, seed):
    """The parameter values FastTD3.__init__ produces (fasttd3.py:80-85): same torch modules, same construction order, same seed.
    Returns (policy, q1, q2) as lists of (weight, bias)."""
    torch.manual_seed(seed)
    pol = _mlp(obs, POLICY_WIDTHS, act)
    torch.nn.init.normal_(pol[-1].weight, 0.0, 0.01)
    torch.nn.init.constant_(pol[-1].bias, 0.0)
    grab = lambda layers: [(l.weight.detach().clone(), l.bias.detach().clone()) for l in layers]
    q1, q2 = grab(_mlp(obs + act, Q_WIDTHS, nr_atoms)), grab(_mlp(obs + act, Q_WIDTHS, nr_atoms))
    _mlp(obs + act, Q_WIDTHS, nr_atoms), _mlp(obs + act, Q_WIDTHS, nr_atoms)   # the targets consume the generator before being overwritten
    return grab(pol), q1, q2


def leaves(net):
    return [t for wb in net for t in wb]


def _clone(net, grad):
    f = (lambda t: t.clone().requires_grad_(True)) if grad else (lambda t: t.clone())
    return [(f(w), f(b)) for w, b in net]


def mlp_forward(net, x):
    for w, b in net[:-1]:
        x = F.relu(F.linear(x, w, b))
    return F.linear(x, *net[-1])


def policy_forward(pol, x):
    return torch.tanh(mlp_forward(pol, x))


def q_forward(q, x, a):
    return mlp_forward(q, torch.cat([x, a], dim=1))


def act(pol, x, noise=None, noise_scales=None, low=None, high=None, clip_rescale=False):
    """Policy.get_action (policy.py:57-66): (action, processed_action)."""
    with torch.no_grad():
        action = policy_forward(pol, x)
        if noise is not None:
            action = action + noise * noise_scales
        processed = action
        if clip_rescale:
            processed = low + 0.5 * (torch.clamp(action, -1.0, 1.0) + 1.0) * (high - low)
    return action, processed


class Learner:
    def __init__(self, pol, q1, q2, lr, weight_decay, gamma, tau, v_min, v_max, nr_atoms, smoothing_epsilon, smoothing_clip_value,
                 clipped_double_q=True, max_grad_norm=-1.0):
        self.clipped, self.max_grad_norm = clipped_double_q, max_grad_norm
        self.pol, self.q1, self.q2 = _clone(pol, True), _clone(q1, True), _clone(q2, True)
        self.q1t, self.q2t = _clone(q1, False), _clone(q2, False)
        self.popt = torch.optim.AdamW(leaves(self.pol), lr=lr, weight_decay=weight_decay)
        self.qopt = torch.optim.AdamW(leaves(self.q1) + leaves(self.q2), lr=lr, weight_decay=weight_decay)
        self.gamma, self.tau, self.v_min, self.v_max, self.nr_atoms = gamma, tau, v_min, v_max, nr_atoms
        self.se, self.sclip = smoothing_epsilon, smoothing_clip_value
        self.support = torch.linspace(v_min, v_max, nr_atoms)

    def set_lr(self, lr):
        for opt in (self.popt, self.qopt):
            for g in opt.param_groups:
                g["lr"] = lr

    def critic_step(self, s, ns, a, r, dones, truncs, eff, smoothing_noise):
        """fasttd3.py:139-225, then the polyak update of :316-320."""
        with torch.no_grad():
            noise = torch.clamp(smoothing_noise * self.se, -self.sclip, self.sclip)
            na = torch.clamp(policy_forward(self.pol, ns) + noise, -1.0, 1.0)
            delta_z = (self.v_max - self.v_min) / (self.nr_atoms - 1)
            bootstrap = 1.0 - (dones * (1.0 - truncs))
            discount = (self.gamma ** eff) * bootstrap
            target_z = torch.clamp(r.unsqueeze(1) + discount.unsqueeze(1) * self.support.unsqueeze(0), self.v_min, self.v_max)
            b = (target_z - self.v_min) / delta_z
            lo0, up0 = torch.floor(b).long(), torch.ceil(b).long()
            is_int = lo0 == up0
            lo = torch.where(is_int & (lo0 > 0), lo0 - 1, lo0)
            up = torch.where(is_int & (lo0 == 0), up0 + 1, up0)
            d1 = F.softmax(q_forward(self.q1t, ns, na), dim=1)
            d2 = F.softmax(q_forward(self.q2t, ns, na), dim=1)
            wl, wu = up.float() - b, b - lo.float()
            proj1, proj2 = torch.zeros_like(d1), torch.zeros_like(d2)
            for proj, d in ((proj1, d1), (proj2, d2)):
                proj.scatter_add_(1, lo, d * wl)
                proj.scatter_add_(1, up, d * wu)
            q1_next_value = (proj1 * self.support).sum(1)
            if self.clipped:
                q2_next_value = (proj2 * self.support).sum(1)
                proj1 = proj2 = torch.where(q1_next_value.unsqueeze(1) < q2_next_value.unsqueeze(1), proj1, proj2)
        l1 = -(proj1 * F.log_softmax(q_forward(self.q1, s, a), dim=1)).sum(1).mean()
        l2 = -(proj2 * F.log_softmax(q_forward(self.q2, s, a), dim=1)).sum(1).mean()
        q_loss = l1 + l2
        self.qopt.zero_grad()
        q_loss.backward()
        params = leaves(self.q1) + leaves(self.q2)
        if self.max_grad_norm != -1.0:
            cg = float(torch.nn.utils.clip_grad_norm_(params, self.max_grad_norm))
        else:
            cg = math.sqrt(sum(float(p.grad.norm(2) ** 2) for p in params))
        self.qopt.step()
        with torch.no_grad():
            for tgt, src in ((self.q1t, self.q1), (self.q2t, self.q2)):
                for pt, ps in zip(leaves(tgt), leaves(src)):
                    pt.mul_(1.0 - self.tau).add_(ps.detach(), alpha=self.tau)
        return {"loss/q_loss": q_loss.item(), "q/q_min": q1_next_value.min().item(), "q/q_max": q1_next_value.max().item(),
                "gradients/critic_grad_norm": cg}

    def policy_step(self, s):
        """fasttd3.py:104-136."""
        a = policy_forward(self.pol, s)
        v1 = (F.softmax(q_forward(self.q1, s, a), dim=1) * self.support).sum(1)
        v2 = (F.softmax(q_forward(self.q2, s, a), dim=1) * self.support).sum(1)
        qv = torch.minimum(v1, v2) if self.clipped else (v1 + v2) / 2.0
        loss = -qv.mean()
        self.popt.zero_grad()
        for p in leaves(self.q1) + leaves(self.q2):
            p.grad = None
        loss.backward()
        if self.max_grad_norm != -1.0:
            pg = float(torch.nn.utils.clip_grad_norm_(leaves(self.pol), self.max_grad_norm))
        else:
            pg = math.sqrt(sum(float(p.grad.norm(2) ** 2) for p in leaves(self.pol)))
        self.popt.step()
        return {"loss/policy_loss": loss.item(), "gradients/policy_grad_norm": pg}
