"""TEST INFRASTRUCTURE ONLY -- CPU (torch fp32) restatement of the rsl_rl update path.

Restates, functionally over a flat ``{name: tensor}`` parameter dict that uses the
reference's ``state_dict`` names:

* ``RolloutStorage.compute_returns``      rsl_rl/rsl_rl/storage/rollout_storage.py:136-150  (RS)
* ``PPO.process_env_step`` reward path    rsl_rl/rsl_rl/algorithms/ppo.py:129-134           (PPO)
* ``ActorCritic`` forward / log-prob / entropy   rsl_rl/rsl_rl/modules/actor_critic.py:39-353 (AC)
* ``PPO.update`` / ``update_dagger`` / ``enforce_min_std``   PPO:152-296
* ``torch.optim.Adam`` single-tensor step and ``clip_grad_norm_`` as called at PPO:243-246
  (torch library code, restated from its documented algorithm).

Backward passes use torch.autograd on CPU (this is the floating-point oracle the brief
allows); the CUDA kernels implement the backward by hand and are compared against it.

PINNING: tests/golden/make_golden.py executes the unmodified reference classes
(`/root/reference/rsl_rl`) on the same inputs and asserts this module reproduces returns,
advantages, mean losses, clipped gradients and post-Adam parameters; vectors are committed
under tests/golden/.  Only tests/, __graft_entry__.smoke() and bench.py (cpu_baseline /
--impl reference) may import this module; the product path never does.
"""
from __future__ import annotations

import math
from typing import Dict, List

import torch
import torch.nn.functional as F

# parameter manifest in `ActorCritic.parameters()` order (std first: it is registered on the
# root module, AC:296; children follow in construction order AC:186-288)
def param_manifest(num_prop=76, num_priv=24, num_hist=10, priv_dims=(64, 20), actor_dims=(128,),
                   critic_dims=(128,), leg_dims=(128, 128), arm_dims=(128, 128), n_leg=12, n_arm=6):
    m = [("std", (1, n_leg + n_arm))]

    def lin(prefix, idx, o, i):
        m.append((f"{prefix}.{idx}.weight", (o, i)))
        m.append((f"{prefix}.{idx}.bias", (o,)))

    d = num_priv
    for k, o in enumerate(priv_dims):
        lin("actor.priv_encoder", 2 * k, o, d)
        d = o
    latent = d
    assert num_hist == 10, "only the tsteps==10 history encoder (AC:57-62) is restated"
    lin("actor.history_encoder.encoder", 0, 30, num_prop)
    m += [("actor.history_encoder.conv_layers.0.weight", (20, 30, 4)), ("actor.history_encoder.conv_layers.0.bias", (20,)),
          ("actor.history_encoder.conv_layers.2.weight", (10, 20, 2)), ("actor.history_encoder.conv_layers.2.bias", (10,))]
    lin("actor.history_encoder.linear_output", 0, latent, 30)
    d = num_prop + latent
    for k, o in enumerate(actor_dims):
        lin("actor.actor_backbone", 2 * k, o, d)
        d = o
    for head, dims, n_out in (("actor.actor_leg_control_head", leg_dims, n_leg), ("actor.actor_arm_control_head", arm_dims, n_arm)):
        dd = d
        for k, o in enumerate(list(dims) + [n_out]):
            lin(head, 2 * k, o, dd)
            dd = o
    d = num_prop + num_priv
    for k, o in enumerate(critic_dims):
        lin("critic.critic_backbone", 2 * k, o, d)
        d = o
    for head, dims in (("critic.critic_leg_control_head", leg_dims), ("critic.critic_arm_control_head", arm_dims)):
        dd = d
        for k, o in enumerate(list(dims) + [1]):
            lin(head, 2 * k, o, dd)
            dd = o
    return m


def _mlp(P, prefix, x, n_layers, last_act):
    """Sequential of Linear(+ELU) blocks named prefix.{0,2,4..}; `last_act` in {elu,tanh,None}."""
    for k in range(n_layers):
        x = F.linear(x, P[f"{prefix}.{2 * k}.weight"], P[f"{prefix}.{2 * k}.bias"])
        if k < n_layers - 1:
            x = F.elu(x)
        elif last_act == "elu":
            x = F.elu(x)
        elif last_act == "tanh":
            x = torch.tanh(x)
    return x


def _count(P, prefix):
    k = 0
    while f"{prefix}.{2 * k}.weight" in P:
        k += 1
    return k


def priv_latent(P, obs, num_prop=76, num_priv=24):
    return _mlp(P, "actor.priv_encoder", obs[:, num_prop:num_prop + num_priv], _count(P, "actor.priv_encoder"), "elu")  # AC:219-221


def hist_latent(P, obs, num_prop=76, num_hist=10):
    h = obs[:, -num_hist * num_prop:].reshape(-1, num_hist, num_prop)                       # AC:223-225
    nd = h.shape[0]
    pre = "actor.history_encoder"
    proj = F.elu(F.linear(h.reshape(nd * num_hist, -1), P[pre + ".encoder.0.weight"], P[pre + ".encoder.0.bias"]))  # AC:80
    x = proj.reshape(nd, num_hist, -1).permute(0, 2, 1)
    x = F.elu(F.conv1d(x, P[pre + ".conv_layers.0.weight"], P[pre + ".conv_layers.0.bias"], stride=2))            # AC:59
    x = F.elu(F.conv1d(x, P[pre + ".conv_layers.2.weight"], P[pre + ".conv_layers.2.bias"], stride=1))            # AC:60
    x = x.flatten(1)
    return F.elu(F.linear(x, P[pre + ".linear_output.0.weight"], P[pre + ".linear_output.0.bias"]))               # AC:72


def actor_mean(P, obs, hist_encoding=False, num_prop=76, num_priv=24, num_hist=10):
    z = hist_latent(P, obs, num_prop, num_hist) if hist_encoding else priv_latent(P, obs, num_prop, num_priv)       # AC:204-217
    h = _mlp(P, "actor.actor_backbone", torch.cat([obs[:, :num_prop], z], dim=1), _count(P, "actor.actor_backbone"), "elu")
    leg = _mlp(P, "actor.actor_leg_control_head", h, _count(P, "actor.actor_leg_control_head"), "tanh")
    arm = _mlp(P, "actor.actor_arm_control_head", h, _count(P, "actor.actor_arm_control_head"), "tanh")
    return torch.cat([leg, arm], dim=-1)


def critic_values(P, obs, num_prop=76, num_priv=24):
    h = _mlp(P, "critic.critic_backbone", obs[:, :num_prop + num_priv], _count(P, "critic.critic_backbone"), "elu")  # AC:280-286
    leg = _mlp(P, "critic.critic_leg_control_head", h, _count(P, "critic.critic_leg_control_head"), None)
    arm = _mlp(P, "critic.critic_arm_control_head", h, _count(P, "critic.critic_arm_control_head"), None)
    return torch.cat([leg, arm], dim=-1)


def log_prob2(mean, std, actions, n_leg=12):
    """Diagonal-Gaussian log-prob summed per group -> [B,2] (AC:341-345 over torch Normal)."""
    sigma = mean * 0.0 + std                                                                # AC:333-335
    lp = -((actions - mean) ** 2) / (2 * sigma ** 2) - sigma.log() - math.log(math.sqrt(2 * math.pi))
    return torch.cat([lp[:, :n_leg].sum(-1, keepdim=True), lp[:, n_leg:].sum(-1, keepdim=True)], dim=-1)


def entropy2(mean, std, n_leg=12):
    sigma = mean * 0.0 + std
    ent = 0.5 + 0.5 * math.log(2 * math.pi) + torch.log(sigma)                              # AC:326-331
    return torch.cat([ent[:, :n_leg].sum(-1, keepdim=True), ent[:, n_leg:].sum(-1, keepdim=True)], dim=-1)


def policy_act(P, obs, eps, hist_encoding=False):
    """PPO.act (PPO:115-127) with the standard-normal draw `eps` supplied by the caller."""
    with torch.no_grad():
        mean = actor_mean(P, obs, hist_encoding)
        sigma = mean * 0.0 + P["std"]
        actions = mean + sigma * eps
        return dict(actions=actions, values=critic_values(P, obs), log_prob=log_prob2(mean, P["std"], actions),
                    mean=mean, sigma=sigma)


def bootstrap_rewards(rew, arm_rew, values, time_outs, gamma):
    r = torch.stack([rew.clone(), arm_rew.clone()], dim=-1)                                 # PPO:130
    return r + gamma * torch.squeeze(values * time_outs.unsqueeze(1), 1)                    # PPO:133-134


def compute_returns(rewards, values, dones, last_values, gamma, lam):
    """RS:136-150.  rewards/values [T,N,2], dones [T,N,1] uint8, last_values [N,2]."""
    T = rewards.shape[0]
    returns = torch.zeros_like(values)
    adv = 0
    for t in reversed(range(T)):
        nxt = last_values if t == T - 1 else values[t + 1]
        not_term = 1.0 - dones[t].float()
        delta = rewards[t] + not_term * gamma * nxt - values[t]
        adv = delta + not_term * gamma * lam * adv
        returns[t] = adv + values[t]
    a = returns - values
    a = (a - a.mean()) / (a.std() + 1e-8)
    return returns, a


class Adam:
    """torch.optim.Adam(lr, betas=(0.9,0.999), eps=1e-8, weight_decay=0) single-tensor step.
    Parameters whose grad is None are skipped and keep their own step count."""

    def __init__(self, names, lr, betas=(0.9, 0.999), eps=1e-8):
        self.names, self.lr, self.b1, self.b2, self.eps = list(names), lr, betas[0], betas[1], eps
        self.state: Dict[str, dict] = {}

    def step(self, P, G):
        for n in self.names:
            g = G.get(n)
            if g is None:
                continue
            st = self.state.setdefault(n, dict(step=0, m=torch.zeros_like(P[n]), v=torch.zeros_like(P[n])))
            st["step"] += 1
            st["m"].mul_(self.b1).add_(g, alpha=1 - self.b1)
            st["v"].mul_(self.b2).addcmul_(g, g, value=1 - self.b2)
            bc1 = 1 - self.b1 ** st["step"]
            bc2 = 1 - self.b2 ** st["step"]
            denom = (st["v"].sqrt() / math.sqrt(bc2)).add_(self.eps)
            P[n].addcdiv_(st["m"], denom, value=-(self.lr / bc1))


def clip_grad_norm(G: Dict[str, torch.Tensor], names, max_norm):
    gs = [G[n] for n in names if G.get(n) is not None]
    total = torch.norm(torch.stack([torch.norm(g, 2.0) for g in gs]), 2.0)
    coef = torch.clamp(max_norm / (total + 1e-6), max=1.0)
    for g in gs:
        g.mul_(coef)
    return total


HIST_PREFIX = "actor.history_encoder."


def value_mixing_ratio(counter, sched):
    return min(max((counter - sched[1]) / sched[2], 0), 1) * sched[0]                       # PPO:301-302


def priv_reg_coef(counter, sched):
    stage = min(max((counter - sched[2]), 0) / sched[3], 1)                                 # PPO:178
    return stage * (sched[1] - sched[0]) + sched[0]                                         # PPO:179


def torque_supervision_weight(counter, sched):
    return (1 - min(max((counter - sched[1]) / sched[2], 0), 1)) * sched[0]                 # PPO:304-305


def arm_fk_fixed_gains(coefs, target_arm_dof_pos, current_arm_dof_pos, current_arm_dof_vel):
    """PPO:318-323.  coefs = (default_arm_p_gains, default_arm_d_gains, default_arm_dof_pos) of PPO:307-310."""
    kp, kd, q0 = coefs
    return kp * (target_arm_dof_pos + q0 - current_arm_dof_pos) - kd * current_arm_dof_vel


def minibatch_loss(P, mb, hp, counter):
    """Loss of one PPO mini-batch (PPO:166-239).  mb: dict of gathered rows.  hp["torque_supervision"] (with
    hp["adaptive_arm_gains"] False) adds the arm torque-supervision term PPO:224-239; hp["arm_coefs"] = the three tensors of PPO:307-310."""
    obs = mb["obs"]
    mean = actor_mean(P, obs, False)
    logp = log_prob2(mean, P["std"], mb["actions"])
    value = critic_values(P, obs)
    ent = entropy2(mean, P["std"])
    zp = priv_latent(P, obs)
    with torch.no_grad():
        zh = hist_latent(P, obs)
    reg = (zp - zh.detach()).norm(p=2, dim=1).mean()
    rho = value_mixing_ratio(counter, hp["mixing_schedule"])
    adv = mb["advantages"]
    mix = torch.zeros_like(adv)
    mix[..., 0] = adv[..., 0] + rho * adv[..., 1]
    mix[..., 1] = adv[..., 1] + rho * adv[..., 0]
    ratio = torch.exp(logp - mb["old_log_prob"])
    clip = hp["clip_param"]
    surr = torch.max(-mix * ratio, -mix * torch.clamp(ratio, 1.0 - clip, 1.0 + clip)).mean()
    if hp.get("use_clipped_value_loss", True):
        vclip = mb["values"] + (value - mb["values"]).clamp(-clip, clip)
        vloss = torch.max((value - mb["returns"]).pow(2), (vclip - mb["returns"]).pow(2)).mean()
    else:
        vloss = (mb["returns"] - value).pow(2).mean()
    creg = priv_reg_coef(counter, hp["priv_reg_coef_schedual"])
    loss = surr + hp["value_loss_coef"] * vloss - hp["entropy_coef"] * ent.mean() + creg * reg
    info = dict(surrogate=surr.detach(), value=vloss.detach(), priv_reg=reg.detach(), entropy=ent.mean().detach(), priv_reg_coef=creg,
                mixing_ratio=rho)
    if hp.get("torque_supervision", False):
        assert not hp.get("adaptive_arm_gains", False), "only the fixed-gain branch (PPO:229-231, 318-323) is restated"
        n_arm = mb["target_arm_torques"].shape[-1]
        target_arm_dof_pos = actor_mean(P, obs, False)[:, -n_arm:]                          # PPO:230 act_inference(obs)[:, -6:] (same values as `mean`)
        tau = arm_fk_fixed_gains(hp["arm_coefs"], target_arm_dof_pos, mb["current_arm_dof_pos"], mb["current_arm_dof_vel"])   # PPO:235
        tloss = (tau - mb["target_arm_torques"]).pow(2).mean()                              # PPO:236
        w = torque_supervision_weight(counter, hp["torque_supervision_schedule"])           # PPO:237
        loss = loss + tloss * w                                                             # PPO:238
        info.update(arm_torques=tloss.detach(), torque_supervision_weight=w)
    return loss, info


def gather(storage, idx):
    f = lambda x: x.flatten(0, 1)[idx]  # noqa: E731                                        RS:165-201
    mb = dict(obs=f(storage["observations"]), actions=f(storage["actions"]), values=f(storage["values"]),
              returns=f(storage["returns"]), old_log_prob=f(storage["actions_log_prob"]),
              advantages=f(storage["advantages"]))
    for k in ("target_arm_torques", "current_arm_dof_pos", "current_arm_dof_vel"):           # RS:178-180,199-201
        if k in storage:
            mb[k] = f(storage[k])
    return mb


def ppo_update(P, opt: Adam, storage, indices, hp, counter, record=None):
    """PPO.update (PPO:152-263) given the permutation `indices` the generator drew (RS:163)."""
    names = list(P.keys())
    nmb, nep = hp["num_mini_batches"], hp["num_learning_epochs"]
    mbs = indices.numel() // nmb
    logs: List[dict] = []
    for ep in range(nep):
        for i in range(nmb):
            mb = gather(storage, indices[i * mbs:(i + 1) * mbs])
            for n in names:
                P[n].requires_grad_(True)
                P[n].grad = None
            loss, info = minibatch_loss(P, mb, hp, counter)
            loss.backward()
            G = {n: (P[n].grad.detach() if P[n].grad is not None else None) for n in names}
            for n in names:
                P[n].requires_grad_(False)
            info["grad_norm"] = clip_grad_norm(G, names, hp["max_grad_norm"])
            if record is not None:
                record(len(logs), P, G, "pre_step")
            with torch.no_grad():
                opt.step(P, G)
            if record is not None:
                record(len(logs), P, G, "post_step")
            logs.append(info)
    if hp.get("min_policy_std") is not None:                                                # PPO:293-296
        P["std"] = torch.max(P["std"], torch.tensor(hp["min_policy_std"]))
    return logs


def dagger_update(P, opt: Adam, storage, indices, hp):
    """PPO.update_dagger (PPO:265-291): hist-encoder regression onto the detached priv latent."""
    names = [n for n in P if n.startswith(HIST_PREFIX)]
    nmb, nep = hp["num_mini_batches"], hp["num_learning_epochs"]
    mbs = indices.numel() // nmb
    losses = []
    for ep in range(nep):
        for i in range(nmb):
            obs = storage["observations"].flatten(0, 1)[indices[i * mbs:(i + 1) * mbs]]
            for n in names:
                P[n].requires_grad_(True)
                P[n].grad = None
            with torch.no_grad():
                zp = priv_latent(P, obs)
            zh = hist_latent(P, obs)
            loss = (zp.detach() - zh).norm(p=2, dim=1).mean()
            loss.backward()
            G = {n: P[n].grad.detach() for n in names}
            for n in names:
                P[n].requires_grad_(False)
            clip_grad_norm(G, names, hp["max_grad_norm"])
            with torch.no_grad():
                opt.step(P, G)
            losses.append(loss.detach())
    return losses
