"""CPU oracle of FastTD3 with observation index sets - TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A thin layer over oracle/fasttd3_oracle.py, which it leaves unchanged: the reference index-selects each network's input before its first
layer (rl_x/algorithms/fasttd3/pytorch/policy.py:52 `x = x[..., self.policy_observation_indices]`, q_network.py:39 then
`cat([x, a])`), so the policy here sees `x[..., policy_idx]` and the Q networks `[x[..., critic_idx] | a]`; None = every column.  The
Learner of the oracle calls the module's `policy_forward` / `q_forward`; this layer's Learner runs its steps with those two names bound
to the selecting versions and restores them afterwards.  Pinned against the executed reference by tests/golden/fasttd3_obs_indices.npz
(tests/golden/make_golden_fasttd3_obs_indices.py).
"""
import contextlib

import torch

from oracle import fasttd3_oracle as TD

_policy_forward, _q_forward = TD.policy_forward, TD.q_forward


def select(x, idx):
    return x if idx is None else x[..., torch.as_tensor(idx, dtype=torch.long, device=x.device)]


def reference_init(obs, act, nr_atoms, seed, policy_idx=None, critic_idx=None):
    """fasttd3_oracle.reference_init with the fan-ins P = len(policy_idx) and C + act, C = len(critic_idx) (policy.py:30, q_network.py:24):
    the same modules in the same order under the same seed."""
    P = obs if policy_idx is None else len(policy_idx)
    C = obs if critic_idx is None else len(critic_idx)
    torch.manual_seed(seed)
    pol = TD._mlp(P, TD.POLICY_WIDTHS, act)
    torch.nn.init.normal_(pol[-1].weight, 0.0, 0.01)
    torch.nn.init.constant_(pol[-1].bias, 0.0)
    grab = lambda layers: [(l.weight.detach().clone(), l.bias.detach().clone()) for l in layers]
    q1, q2 = grab(TD._mlp(C + act, TD.Q_WIDTHS, nr_atoms)), grab(TD._mlp(C + act, TD.Q_WIDTHS, nr_atoms))
    TD._mlp(C + act, TD.Q_WIDTHS, nr_atoms), TD._mlp(C + act, TD.Q_WIDTHS, nr_atoms)   # the targets consume the generator too
    return grab(pol), q1, q2


def policy_forward(pol, x, policy_idx=None):
    return _policy_forward(pol, select(x, policy_idx))


def q_forward(q, x, a, critic_idx=None):
    return _q_forward(q, select(x, critic_idx), a)


def act(pol, x, noise=None, noise_scales=None, low=None, high=None, clip_rescale=False, policy_idx=None):
    return TD.act(pol, select(x, policy_idx), noise, noise_scales, low, high, clip_rescale)


@contextlib.contextmanager
def selecting(policy_idx, critic_idx):
    """TD.policy_forward / TD.q_forward read the selected columns inside the block."""
    TD.policy_forward = lambda pol, x: _policy_forward(pol, select(x, policy_idx))
    TD.q_forward = lambda q, x, a: _q_forward(q, select(x, critic_idx), a)
    try:
        yield
    finally:
        TD.policy_forward, TD.q_forward = _policy_forward, _q_forward


class Learner(TD.Learner):
    """fasttd3_oracle.Learner whose policy reads states[:, policy_idx] and Q networks [states[:, critic_idx] | actions] (fasttd3.py:104-225)."""

    def __init__(self, pol, q1, q2, *args, policy_idx=None, critic_idx=None, **kw):
        super().__init__(pol, q1, q2, *args, **kw)
        self.policy_idx, self.critic_idx = policy_idx, critic_idx

    def critic_step(self, *args):
        with selecting(self.policy_idx, self.critic_idx):
            return super().critic_step(*args)

    def policy_step(self, s):
        with selecting(self.policy_idx, self.critic_idx):
            return super().policy_step(s)
