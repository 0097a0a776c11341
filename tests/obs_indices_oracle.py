"""CPU oracle of PPO and ESPO with observation index sets - TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A thin layer over oracle/ppo_oracle.py and oracle/espo_oracle.py, which it leaves unchanged: the reference index-selects each net's input
before its first layer (rl_x/algorithms/ppo/pytorch/policy.py:62 `x = x[..., self.policy_observation_indices]`, critic.py:45), so the
policy functions here see `x[..., policy_idx]` and the critic functions `x[..., critic_idx]`; None = every column.  Pinned against the
executed reference by tests/golden/ppo_obs_indices.npz (tests/golden/make_golden_ppo_obs_indices.py).
"""
import math

import torch

from oracle import espo_oracle as E
from oracle import ppo_oracle as O


def select(x, idx):
    return x if idx is None else x[..., torch.as_tensor(idx, dtype=torch.long)]


def init_params(obs_dim, act_dim, hidden, std_dev=1.0, seed=0, policy_idx=None, critic_idx=None):
    """ppo_oracle.init_params with P = len(policy_idx) policy inputs and C = len(critic_idx) critic inputs (policy.py:37, critic.py:27)."""
    g = torch.Generator().manual_seed(seed)
    P = obs_dim if policy_idx is None else len(policy_idx)
    C = obs_dim if critic_idx is None else len(critic_idx)

    def lin(out_f, in_f, gain):
        w = torch.empty(out_f, in_f)
        torch.nn.init.orthogonal_(w, gain, generator=g)
        return w, torch.zeros(out_f)

    pol, cri = {}, {}
    for i, (o, inp, gain) in zip((0, 2, 4), ((hidden, P, math.sqrt(2)), (hidden, hidden, math.sqrt(2)), (act_dim, hidden, 0.01))):
        pol[f"policy_mean.{i}.weight"], pol[f"policy_mean.{i}.bias"] = lin(o, inp, gain)
    pol["policy_logstd"] = torch.full((1, act_dim), math.log(std_dev))
    for i, (o, inp, gain) in zip((0, 2, 4), ((hidden, C, math.sqrt(2)), (hidden, hidden, math.sqrt(2)), (1, hidden, 1.0))):
        cri[f"critic.{i}.weight"], cri[f"critic.{i}.bias"] = lin(o, inp, gain)
    return pol, cri


def policy_mean(pol, x, policy_idx=None):
    return O.policy_mean(pol, select(x, policy_idx))


def critic_value(cri, x, critic_idx=None):
    return O.critic_value(cri, select(x, critic_idx))


def get_logprob_entropy(pol, x, action, policy_idx=None):
    return O.get_logprob_entropy(pol, select(x, policy_idx), action)


def get_action_logprob(pol, x, noise, act_low, act_high, clip_rescale=True, policy_idx=None):
    return O.get_action_logprob(pol, select(x, policy_idx), noise, act_low, act_high, clip_rescale)


def get_deterministic_action(pol, x, act_low, act_high, clip_rescale=True, policy_idx=None):
    return O.get_deterministic_action(pol, select(x, policy_idx), act_low, act_high, clip_rescale)


class Learner(O.Learner):
    """ppo_oracle.Learner whose policy loss sees states[:, policy_idx] and critic loss states[:, critic_idx] (ppo.py:121-166)."""

    def __init__(self, pol, cri, policy_idx=None, critic_idx=None, **kw):
        super().__init__(pol, cri, **kw)
        self.policy_idx, self.critic_idx = policy_idx, critic_idx

    def grads(self, states, actions, log_probs, advantages, returns):
        self.popt.zero_grad()
        self.copt.zero_grad()
        loss, pg, ent, kl, cf = O.policy_loss(self.pol, select(states, self.policy_idx), actions, log_probs, advantages, self.clip_range,
                                              self.entropy_coef)
        loss.backward()
        closs = O.critic_loss(self.cri, select(states, self.critic_idx), returns, self.critic_coef)
        closs.backward()
        gp = {k: self.pol[k].grad.clone() for k in O.POLICY_KEYS}
        gc = {k: self.cri[k].grad.clone() for k in O.CRITIC_KEYS}
        return gp, gc, dict(pg_loss=pg.item(), critic_loss=closs.item(), entropy_loss=ent.item(), approx_kl=kl.item(), clip_fraction=cf.item())

    def minibatch_step(self, states, actions, log_probs, advantages, returns):
        self.popt.zero_grad()
        with O.autocast_bf16(self.bf16):
            loss, pg, ent, kl, cf = O.policy_loss(self.pol, select(states, self.policy_idx), actions, log_probs, advantages, self.clip_range,
                                                  self.entropy_coef)
        loss.backward()
        pnorm = torch.nn.utils.clip_grad_norm_([self.pol[k] for k in O.POLICY_KEYS], self.max_grad_norm)
        self.popt.step()
        self.copt.zero_grad()
        with O.autocast_bf16(self.bf16):
            closs = O.critic_loss(self.cri, select(states, self.critic_idx), returns, self.critic_coef)
        closs.backward()
        cnorm = torch.nn.utils.clip_grad_norm_([self.cri[k] for k in O.CRITIC_KEYS], self.max_grad_norm)
        self.copt.step()
        return dict(pg_loss=pg.item(), critic_loss=closs.item(), entropy_loss=ent.item(), approx_kl=kl.item(),
                    clip_fraction=cf.item(), policy_grad_norm=pnorm.item(), critic_grad_norm=cnorm.item())


class EspoLearner(E.Learner):
    """espo_oracle.Learner with the same input selection (ESPO's networks are PPO's, espo.py:84-92)."""

    def __init__(self, pol, cri, policy_idx=None, critic_idx=None, **kw):
        super().__init__(pol, cri, **kw)
        self.policy_idx, self.critic_idx = policy_idx, critic_idx

    def minibatch_step(self, states, actions, log_probs, advantages, returns):
        self.popt.zero_grad()
        loss, pg, ent, kl, rd = E.policy_loss(self.pol, select(states, self.policy_idx), actions, log_probs, advantages, self.entropy_coef,
                                              self.delta_op)
        loss.backward()
        pnorm = torch.nn.utils.clip_grad_norm_([self.pol[k] for k in O.POLICY_KEYS], self.max_grad_norm)
        self.popt.step()
        self.copt.zero_grad()
        closs = O.critic_loss(self.cri, select(states, self.critic_idx), returns, self.critic_coef)
        closs.backward()
        cnorm = torch.nn.utils.clip_grad_norm_([self.cri[k] for k in O.CRITIC_KEYS], self.max_grad_norm)
        self.copt.step()
        return dict(pg_loss=pg.item(), critic_loss=closs.item(), entropy_loss=ent.item(), approx_kl=kl.item(), ratio_delta=rd.item(),
                    policy_grad_norm=pnorm.item(), critic_grad_norm=cnorm.item())
