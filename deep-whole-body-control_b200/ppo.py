"""Fused PPO with the reference's method surface (`rsl_rl.algorithms.PPO`,
rsl_rl/rsl_rl/algorithms/ppo.py:38-325, cited PPO:line): `act`, `process_env_step`,
`compute_returns`, `update` (7-tuple), `update_dagger` (float), `enforce_min_std`,
attributes `actor_critic`, `storage`, `learning_rate`, `optimizer`, `counter`.

Every numerical step runs in libdwbc kernels; this class only sequences launches:
  act            -> dwbc_policy_act, writing straight into the storage rows (no RS:95-114 copies)
  process_env_step -> dwbc_store_rewards (time-out bootstrap PPO:133-134) [+ dwbc_track_episodes, OPR:140-154]
  compute_returns  -> dwbc_critic_values + dwbc_gae
  update         -> per mini-batch: dwbc_ppo_minibatch_grad [+ NCCL all-reduce] + dwbc_clip_adam_step
                    (diagnostics=True: dwbc_explained_variance once, dwbc_ppo_minibatch_grad_diag per mini-batch)
  update_dagger  -> per mini-batch: dwbc_dagger_minibatch_grad [+ all-reduce] + dwbc_clip_adam_step

Host<->device synchronisation happens once per update (to return the mean losses), not three
times per mini-batch as in PPO:248-250.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib as L
from . import shard
from .actor_critic import FlatActorCritic
from .graphs import HostUpload
from .storage import FusedRolloutStorage

CHECKPOINT_VERSION = 1          # layout of FusedPPO.state_dict()


# The host arithmetic of the readers of FusedPPO (update(), update_dagger(), episode_buffers(), update_diagnostics()), shared with
# GraphRunner.logs(), which applies it to copies of the same device values taken at the end of each iteration.
def loss_means(sums, num_updates):
    """The mean losses of an update from the sums in `_losses` (surrogate, value, priv-reg, entropy, arm torques).  Evaluated where the
    sums are, on the device in update() and in GraphRunner.logs() alike, so that the two give the same bits."""
    return sums / num_updates


def ppo_result(losses, sched, torque_supervision):
    """update()'s 7-tuple (PPO:263) from the mean losses (a list) and the schedule values _ppo_end returns."""
    value_mixing_ratio, ts_w, priv_reg_coef = sched
    return losses[1], losses[0], (losses[4] if torque_supervision else 0.0), value_mixing_ratio, ts_w, losses[2], priv_reg_coef


def dagger_loss(loss_sum, num_updates):
    """update_dagger()'s mean history-latent loss from the sum in `_losses[0]`."""
    return float(loss_sum) / num_updates


def ring_buffers(ring, pos):
    """OPR's rewbuffer, arm_rewbuffer and lenbuffer (Python float lists, oldest first) from an episode tracker's ring [C, 3] and
    position [2] (next slot, episodes appended since tracking began), both on the host."""
    cap = ring.shape[0]
    n = min(int(pos[1]), cap)
    rows = ring[(int(pos[0]) - n + torch.arange(n)) % cap]
    return dict(rewbuffer=rows[:, 0].tolist(), arm_rewbuffer=rows[:, 1].tolist(), lenbuffer=rows[:, 2].tolist())


def diagnostics_from(d, ev):
    """update_diagnostics()'s dictionary from the per-mini-batch slots d [mini-batches, DIAG_N] and the explained variances ev [2], both
    on the host."""
    d = d.double()
    per = dict(approx_kl=(d[:, L.DIAG_KL_LEG] + d[:, L.DIAG_KL_ARM]).tolist(), approx_kl_leg=d[:, L.DIAG_KL_LEG].tolist(),
               approx_kl_arm=d[:, L.DIAG_KL_ARM].tolist(), clip_fraction_leg=d[:, L.DIAG_CLIP_LEG].tolist(),
               clip_fraction_arm=d[:, L.DIAG_CLIP_ARM].tolist(), grad_norm=d[:, L.DIAG_GRAD_NORM].tolist())
    out = {k: sum(v) / len(v) for k, v in per.items()}
    out.update(grad_norm_max=max(per["grad_norm"]), explained_variance_leg=float(ev[0]), explained_variance_arm=float(ev[1]),
               per_minibatch=per)
    return out


class _AdamState:
    """Flat Adam state of one parameter group; `state_dict()` mimics torch.optim.Adam's layout."""

    def __init__(self, ac: FlatActorCritic, first, count, lr):
        self.ac, self.first, self.count, self.lr = ac, first, count, lr
        self.m = torch.zeros_like(ac.flat)
        self.v = torch.zeros_like(ac.flat)
        self.step = 0
        self.param_groups = [dict(lr=lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0)]

    def _names(self):
        return [n for n in self.ac.offsets if self.first <= self.ac.offsets[n] < self.first + self.count]

    def check_state_dict(self, sd, what):
        """Raise DwbcError unless `sd` is a state_dict() of this group: one entry per parameter, the parameters' shapes, one step."""
        names, shapes = self._names(), dict(self.ac.manifest)
        try:
            params, state = list(sd["param_groups"][0]["params"]), sd["state"]
            if params != list(range(len(names))) or (state and set(state) != set(params)):
                raise L.DwbcError(f"{what}: {len(params)} parameters in the checkpoint, {len(names)} in this optimizer")
            for i, n in enumerate(names):
                if i in state:
                    st = state[i]
                    if tuple(st["exp_avg"].shape) != shapes[n] or tuple(st["exp_avg_sq"].shape) != shapes[n]:
                        raise L.DwbcError(f"{what}: the moments of {n} have shape {tuple(st['exp_avg'].shape)}, not {shapes[n]}")
            if len({int(st["step"]) for st in state.values()}) > 1:
                raise L.DwbcError(f"{what}: the parameters have different step counts")
        except (KeyError, IndexError, TypeError, AttributeError) as e:
            raise L.DwbcError(f"{what}: not an optimizer state_dict ({type(e).__name__}: {e})") from None

    def state_dict(self):
        names = self._names()
        um, uv = self.ac.unflat(self.m), self.ac.unflat(self.v)
        state = {i: dict(step=torch.tensor(float(self.step)), exp_avg=um[n].clone(), exp_avg_sq=uv[n].clone())
                 for i, n in enumerate(names)} if self.step > 0 else {}
        return dict(state=state, param_groups=[dict(self.param_groups[0], params=list(range(len(names))))])

    def load_state_dict(self, sd):
        names = self._names()
        um, uv = self.ac.unflat(self.m), self.ac.unflat(self.v)
        for i, n in enumerate(names):
            if i in sd["state"]:
                um[n].copy_(sd["state"][i]["exp_avg"])
                uv[n].copy_(sd["state"][i]["exp_avg_sq"])
                self.step = int(sd["state"][i]["step"])


class FusedPPO:
    def __init__(self, actor_critic: FlatActorCritic, num_learning_epochs=1, num_mini_batches=1, clip_param=0.2, gamma=0.998,
                 lam=0.95, value_loss_coef=1.0, entropy_coef=0.0, learning_rate=1e-3, max_grad_norm=1.0,
                 use_clipped_value_loss=True, schedule="fixed", desired_kl=0.01, device="cuda:0",
                 mixing_schedule=(0.5, 2000, 4000), torque_supervision=False, torque_supervision_schedule=(0.1, 1000, 1000),
                 adaptive_arm_gains=False, min_policy_std=None, dagger_update_freq=20, priv_reg_coef_schedual=(0, 0, 0, 1),
                 world_size=1, process_group=None, precision="tf32x3", cuda_graphs=False, track_episodes=0,
                 diagnostics=False):
        if adaptive_arm_gains:
            raise L.DwbcError("adaptive_arm_gains (a 12-output arm head, AC:111-125,214-215; off for widowGo1, WGC:168) is not implemented")
        if schedule != "fixed":
            raise L.DwbcError("only schedule='fixed' (WGC:352) is implemented")
        self.device = torch.device(device)
        self.actor_critic = actor_critic
        self.storage = None
        self.learning_rate, self.schedule, self.desired_kl = learning_rate, schedule, desired_kl
        self.clip_param, self.num_learning_epochs, self.num_mini_batches = clip_param, num_learning_epochs, num_mini_batches
        self.value_loss_coef, self.entropy_coef, self.gamma, self.lam = value_loss_coef, entropy_coef, gamma, lam
        self.max_grad_norm, self.use_clipped_value_loss = max_grad_norm, use_clipped_value_loss
        self.min_policy_std = None if min_policy_std is None else torch.tensor(min_policy_std, device=self.device, dtype=torch.float).reshape(-1)
        self.mixing_schedule, self.priv_reg_coef_schedual = list(mixing_schedule), list(priv_reg_coef_schedual)
        # arm torque supervision with fixed gains (PPO:224-239, 318-323): off in the shipped config (WGC:173), on in PPO's own defaults (PPO:57)
        self.torque_supervision, self.adaptive_arm_gains = bool(torque_supervision), False
        self.torque_supervision_schedule = list(torque_supervision_schedule)
        self._arm_coefs = None
        self.dagger_update_freq = dagger_update_freq
        self.counter = 0
        self.world_size, self.process_group = world_size, process_group
        self._zh_all = None
        self._packed = False          # tensor-core weight images in the workspace match the current parameters (rollout reuse)
        self._eps_all, self._eps_valid = None, False
        self.precision = precision
        ac = actor_critic
        self.optimizer = _AdamState(ac, 0, ac.num_params, learning_rate)                  # PPO:75
        hf, hc = ac.hist_range
        self.hist_encoder_optimizer = _AdamState(ac, hf, hc, learning_rate)               # PPO:79
        self.grad = torch.zeros_like(ac.flat)
        self._losses = torch.zeros(5, device=self.device)        # surrogate, value, priv_reg, entropy, arm torques
        self._norm_scratch = torch.zeros(L.NORM_SCRATCH, dtype=torch.float64, device=self.device)
        self._grad_norm = torch.zeros(1, device=self.device)
        self._ws = None
        self._ws_rows = 0
        self._hp = L.PpoHyper()
        self._lib = L.lib()
        self.transition = FusedRolloutStorage.Transition()
        self._eps = None
        self.generator = None
        # cuda_graphs: update() and update_dagger() run as CUDA graphs captured on their first call for a key (graph_key) and replayed
        # afterwards, with the same bits as the eager calls (DESIGN §11)
        if cuda_graphs and world_size > 1:
            raise L.DwbcError("cuda_graphs=True does not capture the multi-GPU all-reduce: use world_size == 1")
        self.cuda_graphs = bool(cuda_graphs)
        self._graphs = {}
        # track_episodes = C > 0: the runner's per-step bookkeeping (OPR:140-154: running returns and lengths, the last C finished
        # episodes) runs on the device inside process_env_step; episode_buffers() reads it once per call (DESIGN §11)
        if isinstance(track_episodes, bool) or not isinstance(track_episodes, int) or track_episodes < 0:
            raise L.DwbcError(f"track_episodes must be a non-negative int (the number of finished episodes kept), not {track_episodes!r}")
        self.track_episodes = track_episodes
        self._episodes = None
        # diagnostics: update() also measures approximate KL, clip fractions, pre-clip gradient norms and explained variance on the device,
        # captured with it; update_diagnostics() reads them once per call (DESIGN §13)
        if not isinstance(diagnostics, bool):
            raise L.DwbcError(f"diagnostics must be True or False, not {diagnostics!r}")
        self.diagnostics = diagnostics
        self._diag, self._diag_steps = None, 0          # [mini-batches, DIAG_N] of the last update(), and how many it ran
        if diagnostics:
            self._diag_ev = torch.zeros(2, device=self.device)                                  # explained variance (leg, arm)
            self._ev_scratch = torch.zeros(L.EV_SCRATCH, dtype=torch.float64, device=self.device)

    # ------------------------------------------------------------------ plumbing
    def init_storage(self, num_envs, num_transitions_per_env, actor_obs_shape, critic_obs_shape, action_shape):
        self.storage = FusedRolloutStorage(num_envs, num_transitions_per_env, actor_obs_shape, critic_obs_shape, action_shape, self.device)
        self._eps = torch.zeros(num_envs, *action_shape, device=self.device)
        self._last_values = torch.zeros(num_envs, 2, device=self.device)
        self._act_tmp = [torch.zeros(num_envs, *action_shape, device=self.device) for _ in range(3)] + \
                        [torch.zeros(num_envs, 2, device=self.device) for _ in range(2)]
        self._workspace(max(num_envs, num_envs * num_transitions_per_env // self.num_mini_batches))
        if self.torque_supervision:
            self.storage.enable_torque_supervision(self.actor_critic.num_arm_actions)
        if self.track_episodes:
            self._episodes = dict(running=torch.zeros(num_envs, 3, device=self.device), ring=torch.zeros(self.track_episodes, 3, device=self.device),
                                  pos=torch.zeros(2, dtype=torch.int64, device=self.device))

    @property
    def precision(self):
        return self._precision

    @precision.setter
    def precision(self, value):
        """'fp32' (CUDA-core GEMMs, parity anchor), 'tf32' (wgmma, truncated 10-bit-mantissa operands) or 'tf32x3' (wgmma,
        error-compensated three-product split: fp32-grade).  Travels to the kernels per call inside DwbcNetCfg.precision."""
        if value not in L.PRECISIONS:
            raise L.DwbcError("precision must be one of " + ", ".join(L.PRECISIONS))
        self._precision = value
        self.actor_critic.net_cfg.precision = L.PRECISIONS[value]
        self._packed = False

    def _set_precision(self):
        self.actor_critic.net_cfg.precision = L.PRECISIONS[self._precision]

    def params_changed(self):
        """Call after writing `actor_critic.flat` from outside (load_state_dict does it): the cached weight images are stale."""
        self._packed = False

    def _workspace(self, rows):
        if self._ws is None or rows > self._ws_rows:
            nbytes = self._lib.dwbc_workspace_bytes(C.addressof(self.actor_critic.net_cfg), rows)
            if nbytes < 0:
                raise L.DwbcError("dwbc_workspace_bytes rejected the network configuration")
            self._ws = torch.zeros(nbytes // 4 + 64, device=self.device)
            self._ws_rows = rows
        return self._ws

    def test_mode(self):
        pass

    def train_mode(self):
        pass

    def set_arm_default_coeffs(self, default_arm_p_gains, default_arm_d_gains, default_arm_dof_pos):
        """PPO:307-310 (called at OPR:91).  Kept as one device tensor [3, n_arm] = p gains, d gains, default positions, each broadcast to
        the arm joints the way PPO:318-323 broadcasts them against the [M, n_arm] batch."""
        self.default_arm_p_gains, self.default_arm_d_gains, self.default_arm_dof_pos = default_arm_p_gains, default_arm_d_gains, default_arm_dof_pos
        if not self.torque_supervision:
            return
        n_arm = self.actor_critic.num_arm_actions
        rows = []
        for x in (default_arm_p_gains, default_arm_d_gains, default_arm_dof_pos):
            x = torch.as_tensor(x, dtype=torch.float, device=self.device)
            if x.dim() > 1 and x.shape[0] != 1:
                raise L.DwbcError("arm coefficients must broadcast to [n_arm] (per-env coefficients are not supported)")
            x = x.reshape(-1) if x.dim() else x
            if x.dim() and x.numel() not in (1, n_arm):
                raise L.DwbcError(f"arm coefficient with {x.numel()} entries does not broadcast to the {n_arm} arm joints (PPO:318-323)")
            rows.append(torch.broadcast_to(x, (n_arm,)))
        self._arm_coefs = torch.stack(rows).contiguous()

    def get_torque_supervision_weight(self):
        sch = self.torque_supervision_schedule
        return (1 - min(max((self.counter - sch[1]) / sch[2], 0), 1)) * sch[0]                   # PPO:304-305

    # ------------------------------------------------------------------ rollout
    def act(self, obs, critic_obs=None, hist_encoding=False, eps=None):
        """PPO:115-127.  Outputs land directly in storage row `storage.step` when a storage exists."""
        ac, s = self.actor_critic, self.storage
        self._set_precision()
        n = obs.shape[0]
        if eps is None:
            na = ac.num_leg_actions + ac.num_arm_actions
            if s is not None and n == s.num_envs and s.step < s.num_transitions_per_env:
                # the standard normals of a whole rollout are drawn by ONE generator launch at its first step (Normal.sample() of AC:337-339
                # draws the same distribution once per step)
                if self._eps_all is None or self._eps_all.shape[:2] != (s.num_transitions_per_env, n):
                    self._eps_all = torch.empty(s.num_transitions_per_env, n, na, device=self.device)
                    self._eps_valid = False
                if s.step == 0 or not self._eps_valid:
                    self._eps_all.normal_(generator=self.generator)
                    self._eps_valid = True
                eps = self._eps_all[s.step]
            else:
                if self._eps is None or self._eps.shape[0] != n:
                    self._eps = torch.empty(n, na, device=self.device)
                eps = self._eps.normal_(generator=self.generator)
        if s is not None and s.step < s.num_transitions_per_env and n == s.num_envs:
            t = s.step
            if obs.data_ptr() != s.observations[t].data_ptr():
                s.observations[t].copy_(obs)                                              # RS:98
            acts, vals, lp, mu, sg = s.actions[t], s.values[t], s.actions_log_prob[t], s.mu[t], s.sigma[t]
            obs_c = s.observations[t]
        else:
            acts, mu, sg, vals, lp = self._act_tmp if n == self._act_tmp[0].shape[0] else \
                [torch.zeros(n, ac.num_leg_actions + ac.num_arm_actions, device=self.device) for _ in range(3)] + \
                [torch.zeros(n, 2, device=self.device) for _ in range(2)]
            obs_c = obs.contiguous()
        ws = self._workspace(n)
        key = (n, int(bool(hist_encoding)), ac.flat._version)
        packed = self._packed and self._packed_key == key
        L.check(self._lib.dwbc_policy_act(C.addressof(ac.net_cfg), L.ptr(ac.flat), L.ptr(obs_c), obs_c.stride(0), L.ptr(eps),
                                          int(bool(hist_encoding)), L.ptr(acts), L.ptr(vals), L.ptr(lp), L.ptr(mu), L.ptr(sg), n,
                                          int(packed), L.ptr(ws), L.stream_ptr()), "dwbc_policy_act")
        self._packed, self._packed_key = True, key
        tr = self.transition
        tr.actions, tr.values, tr.actions_log_prob, tr.action_mean, tr.action_sigma = acts, vals, lp, mu, sg
        tr.observations = tr.critic_observations = obs
        return acts

    def process_env_step(self, rewards, arm_rewards, dones, infos):
        """PPO:129-146 + RS:95-114 (the other transition fields were already written by `act`)."""
        s = self.storage
        if s.step >= s.num_transitions_per_env:
            raise AssertionError("Rollout buffer overflow")                               # RS:96-97
        t = s.step
        stored = infos.get("dwbc_stored_rows") if isinstance(infos, dict) else None
        store = stored is None or stored != (s.rewards[t].data_ptr(), s.dones[t].data_ptr())
        if store or self._episodes is not None:
            d8 = (dones if dones.dtype in (torch.uint8, torch.bool) else (dones != 0)).contiguous()
        if store:
            # (else: the post-physics kernel already wrote this step's rewards / dones rows, FusedWidowGo1Core.set_transition_target)
            to = infos.get("time_outs") if isinstance(infos, dict) else None
            to8 = None if to is None else (to if to.dtype in (torch.uint8, torch.bool) else (to != 0)).contiguous()
            L.check(self._lib.dwbc_store_rewards(L.ptr(rewards.float().contiguous(), torch.float32), L.ptr(arm_rewards.float().contiguous(), torch.float32),
                                                 L.ptr(s.values[t]), L.ptr(to8, (torch.uint8, torch.bool)), L.ptr(d8, (torch.uint8, torch.bool)), self.gamma,
                                                 L.ptr(s.rewards[t]), L.ptr(s.dones[t]), s.num_envs, L.stream_ptr()), "dwbc_store_rewards")
        if self._episodes is not None:
            # the un-bootstrapped rewards env.step returned (OPR:147), not the storage row
            e = self._episodes
            L.check(self._lib.dwbc_track_episodes(L.ptr(rewards.float().contiguous(), torch.float32), L.ptr(arm_rewards.float().contiguous(), torch.float32),
                                                  L.ptr(d8, (torch.uint8, torch.bool)), s.num_envs, L.ptr(e["running"]), L.ptr(e["ring"]),
                                                  L.ptr(e["pos"]), self.track_episodes, L.stream_ptr()), "dwbc_track_episodes")
        if self.torque_supervision and isinstance(infos, dict) and "target_arm_torques" in infos:          # PPO:136-142, RS:108-111
            s.target_arm_torques[t].copy_(infos["target_arm_torques"])
            s.current_arm_dof_pos[t].copy_(infos["current_arm_dof_pos"])
            s.current_arm_dof_vel[t].copy_(infos["current_arm_dof_vel"])
        s.step += 1
        self.transition.clear()

    def compute_returns(self, last_critic_obs):
        """PPO:148-150."""
        ac, s = self.actor_critic, self.storage
        self._set_precision()
        obs = last_critic_obs.contiguous()
        L.check(self._lib.dwbc_critic_values(C.addressof(ac.net_cfg), L.ptr(ac.flat), L.ptr(obs), obs.stride(0),
                                             L.ptr(self._last_values), obs.shape[0], L.ptr(self._workspace(obs.shape[0])),
                                             L.stream_ptr()), "dwbc_critic_values")
        self._packed = False                      # dwbc_critic_values re-packs the critic into the same workspace region
        s.compute_returns(self._last_values, self.gamma, self.lam, self.world_size, self.process_group)

    def episode_buffers(self):
        """OPR's rewbuffer, arm_rewbuffer and lenbuffer (OPR:140-154, maxlen track_episodes) as Python float lists, oldest first: the
        episodes finished since tracking began, read with one synchronisation."""
        if self._episodes is None:
            raise L.DwbcError("episode_buffers() needs FusedPPO(track_episodes=C > 0) and init_storage()")
        ring = self._episodes["ring"].to("cpu", non_blocking=True)
        pos = self._episodes["pos"].to("cpu", non_blocking=True)
        if self.device.type == "cuda":
            torch.cuda.current_stream(self.device).synchronize()
        return ring_buffers(ring, pos)

    def _episodes_shape(self):
        return None if self._episodes is None else (self._episodes["running"].shape[0], self.track_episodes)

    # ------------------------------------------------------------------ schedules (PPO:178-179, 301-302)
    def get_value_mixing_ratio(self):
        return min(max((self.counter - self.mixing_schedule[1]) / self.mixing_schedule[2], 0), 1) * self.mixing_schedule[0]

    def get_priv_reg_coef(self):
        sch = self.priv_reg_coef_schedual
        stage = min(max((self.counter - sch[2]), 0) / sch[3], 1)
        return stage * (sch[1] - sch[0]) + sch[0]

    def _fill_hp(self):
        h = self._hp
        h.clip_param, h.value_loss_coef, h.entropy_coef = self.clip_param, self.value_loss_coef, self.entropy_coef
        h.priv_reg_coef, h.mixing_ratio = self.get_priv_reg_coef(), self.get_value_mixing_ratio()
        h.use_clipped_value_loss = int(self.use_clipped_value_loss)
        h.max_grad_norm, h.lr, h.beta1, h.beta2, h.adam_eps = self.max_grad_norm, self.learning_rate, 0.9, 0.999, 1e-8
        h.grad_scale = shard.grad_scale(self.world_size)
        if self.torque_supervision:
            if self._arm_coefs is None:
                raise L.DwbcError("torque_supervision needs set_arm_default_coeffs() first (OPR:91)")
            h.torque_supervision_weight, h.arm_coefs = self.get_torque_supervision_weight(), self._arm_coefs.data_ptr()
        else:
            h.torque_supervision_weight, h.arm_coefs = 0.0, None
        return h

    def _allreduce(self, first, count):
        shard.allreduce_grad_(self.grad, first, count, self.world_size, self.process_group)

    # ------------------------------------------------------------------ update (PPO:152-263)
    def update(self, indices=None, on_step=None):
        return self._ppo_finish(self._ppo_run(self.cuda_graphs and on_step is None, indices, on_step))

    def _ppo_run(self, graphed, indices=None, on_step=None):
        """Every launch of update(), eager or (graphed) as the replay of its CUDA graph; returns the hyper-parameters they ran with."""
        if graphed:
            return self._update_graphed("ppo", indices)
        ac, s, hp = self.actor_critic, self.storage, self._fill_hp()
        self._set_precision()
        self._packed = False                      # the parameters move (and the workspace is re-used with another row count)
        if indices is None:
            indices, _ = s.draw_indices(self.num_mini_batches, self.generator)
        indices = indices.to(torch.int64).contiguous()
        mbs = indices.numel() // self.num_mini_batches
        ws = self._workspace(mbs)
        self._diag_buffer()
        self._ppo_launches(hp, indices, mbs, ws, on_step)
        return hp

    def _diag_buffer(self):
        """The per-mini-batch diagnostics slots of one update() (diagnostics on), allocated for the current mini-batch count."""
        n = self.num_learning_epochs * self.num_mini_batches
        if self.diagnostics and (self._diag is None or self._diag.shape[0] != n):
            self._diag = torch.zeros(n, L.DIAG_N, device=self.device)
        return self._diag

    def _zh_buffer(self):
        s = self.storage
        total = s.num_envs * s.num_transitions_per_env
        lld = (self.actor_critic.priv_dims[-1] + 3) // 4 * 4
        if self._zh_all is None or self._zh_all.shape[0] != total:
            self._zh_all = torch.zeros(total, lld, device=self.device)
        return self._zh_all

    def _ppo_launches(self, hp, indices, mbs, ws, on_step=None, dev=None):
        """Every launch of one update().  dev = (sched, adam_table) device pointers when capturing: the schedule values and the Adam
        bias correction are then read at run time (row k of the table for mini-batch k), and optimizer.step is left to the caller."""
        ac, s = self.actor_critic, self.storage
        self._losses.zero_()
        k = 0
        # The regulariser target z_hist (PPO:175-176) is detached, so update() never moves the history encoder (zero gradient ->
        # zero Adam step): evaluate it once per storage row instead of once per (epoch, row).
        total = s.num_envs * s.num_transitions_per_env
        zh = self._zh_buffer()
        lld = zh.shape[1]
        obs_flat = s.observations.view(total, -1)
        for r0 in range(0, total, mbs):
            nrow = min(mbs, total - r0)
            L.check(self._lib.dwbc_hist_latent(C.addressof(ac.net_cfg), L.ptr(ac.flat), L.ptr(obs_flat[r0:]), obs_flat.stride(0),
                                               L.ptr(zh[r0:]), lld, nrow, L.ptr(ws), L.stream_ptr()), "dwbc_hist_latent")
        s.set_hist_latent(zh)
        diag = self._diag if self.diagnostics else None
        if diag is not None:
            L.check(self._lib.dwbc_explained_variance(L.ptr(s.values), L.ptr(s.returns), total, L.ptr(self._ev_scratch), L.ptr(self._diag_ev),
                                                      L.stream_ptr()), "dwbc_explained_variance")
        for batch_idx in s.mini_batch_generator(self.num_mini_batches, self.num_learning_epochs, indices):
            if diag is not None:
                L.check(self._lib.dwbc_ppo_minibatch_grad_diag(C.addressof(ac.net_cfg), L.ptr(ac.flat), s.c_struct_ptr(), L.ptr(batch_idx), mbs,
                                                               C.addressof(hp), None if dev is None else dev[0], L.ptr(s.mu), L.ptr(s.sigma),
                                                               L.ptr(self.grad), L.ptr(self._losses), L.ptr(diag[k]), L.ptr(ws), L.stream_ptr()),
                        "dwbc_ppo_minibatch_grad_diag")
            elif dev is None:
                L.check(self._lib.dwbc_ppo_minibatch_grad(C.addressof(ac.net_cfg), L.ptr(ac.flat), s.c_struct_ptr(), L.ptr(batch_idx), mbs,
                                                          C.addressof(hp), L.ptr(self.grad), L.ptr(self._losses), L.ptr(ws), L.stream_ptr()),
                        "dwbc_ppo_minibatch_grad")
            else:
                L.check(self._lib.dwbc_ppo_minibatch_grad_sched(C.addressof(ac.net_cfg), L.ptr(ac.flat), s.c_struct_ptr(), L.ptr(batch_idx),
                                                                mbs, C.addressof(hp), dev[0], L.ptr(self.grad), L.ptr(self._losses), L.ptr(ws),
                                                                L.stream_ptr()), "dwbc_ppo_minibatch_grad_sched")
            self._allreduce(0, ac.num_params)
            if on_step is not None:
                on_step(k, "grad")
            opt = self.optimizer
            norm_out = self._grad_norm if diag is None else diag[k, L.DIAG_GRAD_NORM:]       # the pre-clip norm of step k
            if dev is None:
                opt.step += 1
                L.check(self._lib.dwbc_clip_adam_step(L.ptr(ac.flat), L.ptr(self.grad), L.ptr(opt.m), L.ptr(opt.v), 0, ac.num_params,
                                                      C.addressof(hp), opt.step, L.ptr(self._norm_scratch), L.ptr(norm_out),
                                                      L.stream_ptr()), "dwbc_clip_adam_step")
            else:
                L.check(self._lib.dwbc_clip_adam_step_table(L.ptr(ac.flat), L.ptr(self.grad), L.ptr(opt.m), L.ptr(opt.v), 0, ac.num_params,
                                                            C.addressof(hp), k + 1, dev[1], L.ptr(self._norm_scratch), L.ptr(norm_out),
                                                            L.stream_ptr()), "dwbc_clip_adam_step_table")
            if on_step is not None:
                on_step(k, "step")
            k += 1
        s.set_hist_latent(None)

    def _ppo_finish(self, hp):
        losses = loss_means(self._losses, self.num_learning_epochs * self.num_mini_batches).tolist()      # single sync per update
        sched = self._ppo_end(hp)
        self.last_entropy = losses[3]
        return ppo_result(losses, sched, self.torque_supervision)

    def _ppo_end(self, hp):
        """What _ppo_finish does besides reading the losses, which stay in `_losses` on the device: clear the storage, advance
        `counter`, enforce_min_std().  Returns the host-side schedule values of update()'s 7-tuple (ppo_result's `sched`)."""
        self.storage.clear()
        if self.diagnostics:
            self._diag_steps = self.num_learning_epochs * self.num_mini_batches
        self.counter += 1                                                                 # PPO:259
        self.enforce_min_std()
        ts_w = hp.torque_supervision_weight if self.torque_supervision else 0            # PPO:158
        return hp.mixing_ratio, ts_w, hp.priv_reg_coef

    def update_diagnostics(self):
        """Diagnostics of the last update() (FusedPPO(diagnostics=True)), read with one synchronisation: the means over its mini-batches
        of approx_kl (= approx_kl_leg + approx_kl_arm, the KL rsl_rl's adaptive schedule computes, between the rollout policy and the
        parameters each mini-batch saw), clip_fraction_leg / _arm (share of rows whose ratio the clip cut off), grad_norm (pre-clip) and
        grad_norm_max, the value function's explained_variance_leg / _arm (1 - Var(R - V) / Var(R) over the storage, NaN where Var(R) = 0),
        and under 'per_minibatch' the same per mini-batch, in update order.  With world_size > 1 the values are this rank's own (its rows,
        its parameters; the gradient norm is of the all-reduced gradient).  Not training state: checkpoints do not include them."""
        if not self.diagnostics:
            raise L.DwbcError("update_diagnostics() needs FusedPPO(diagnostics=True)")
        if not self._diag_steps:
            raise L.DwbcError("update_diagnostics(): no update() has run yet")
        d = self._diag.to("cpu", non_blocking=True)
        ev = self._diag_ev.to("cpu", non_blocking=True)
        if self.device.type == "cuda":
            torch.cuda.current_stream(self.device).synchronize()
        return diagnostics_from(d, ev)

    def update_dagger(self, indices=None):
        """PPO:265-291."""
        self._dagger_run(self.cuda_graphs, indices)
        return self._dagger_finish()

    def _dagger_run(self, graphed, indices=None):
        """Every launch of update_dagger(), eager or (graphed) as the replay of its CUDA graph."""
        if graphed:
            self._update_graphed("dagger", indices)
            return
        s, hp = self.storage, self._fill_hp()
        self._set_precision()
        self._packed = False
        if indices is None:
            indices, _ = s.draw_indices(self.num_mini_batches, self.generator)
        indices = indices.to(torch.int64).contiguous()
        mbs = indices.numel() // self.num_mini_batches
        ws = self._workspace(mbs)
        self._dagger_launches(hp, indices, mbs, ws)

    def _dagger_launches(self, hp, indices, mbs, ws, dev=None):
        """Every launch of one update_dagger(); dev as in _ppo_launches (only its Adam table is read)."""
        ac, s = self.actor_critic, self.storage
        self._losses.zero_()
        hf, hc = ac.hist_range
        opt = self.hist_encoder_optimizer
        for k, batch_idx in enumerate(s.mini_batch_generator(self.num_mini_batches, self.num_learning_epochs, indices)):
            L.check(self._lib.dwbc_dagger_minibatch_grad(C.addressof(ac.net_cfg), L.ptr(ac.flat), s.c_struct_ptr(), L.ptr(batch_idx), mbs,
                                                         L.ptr(self.grad), L.ptr(self._losses), L.ptr(ws), L.stream_ptr()),
                    "dwbc_dagger_minibatch_grad")
            self._allreduce(hf, hc)
            if dev is None:
                opt.step += 1
                L.check(self._lib.dwbc_clip_adam_step(L.ptr(ac.flat), L.ptr(self.grad), L.ptr(opt.m), L.ptr(opt.v), hf, hc, C.addressof(hp),
                                                      opt.step, L.ptr(self._norm_scratch), None, L.stream_ptr()), "dwbc_clip_adam_step")
            else:
                L.check(self._lib.dwbc_clip_adam_step_table(L.ptr(ac.flat), L.ptr(self.grad), L.ptr(opt.m), L.ptr(opt.v), hf, hc,
                                                            C.addressof(hp), k + 1, dev[1], L.ptr(self._norm_scratch), None, L.stream_ptr()),
                        "dwbc_clip_adam_step_table")

    def _dagger_finish(self):
        loss = dagger_loss(self._losses[0], self.num_learning_epochs * self.num_mini_batches)
        self._dagger_end()
        return loss

    def _dagger_end(self):
        """What _dagger_finish does besides reading the loss, which stays in `_losses[0]` on the device."""
        self.storage.clear()
        self.counter += 1

    # ------------------------------------------------------------------ CUDA graphs of update() / update_dagger()
    def graph_key(self, kind):
        """What a captured update depends on beyond the per-iteration scalars: a change re-captures.  Storage shape and buffers,
        mini-batching, precision, network and workspace, torque supervision, and the hyper-parameters the launches carry by value."""
        s, ac, h = self.storage, self.actor_critic, self._hp
        key = (kind, s.num_transitions_per_env, s.num_envs, s._obs_all.data_ptr(), self.num_mini_batches, self.num_learning_epochs,
               self._precision, ac.flat.data_ptr(), bytes(ac.net_cfg), self._ws.data_ptr(), self._ws_rows, self.torque_supervision,
               h.clip_param, h.value_loss_coef, h.entropy_coef, h.use_clipped_value_loss, h.max_grad_norm, h.lr, h.beta1, h.beta2,
               h.adam_eps, h.grad_scale, h.arm_coefs)
        if self.diagnostics and kind == "ppo":
            key += (("diagnostics", self._diag_buffer().data_ptr()),)
        return key

    def _update_graphed(self, kind, indices):
        """update() / update_dagger() as one CUDA graph: captured on the first call for a key (graph_key), replayed on later calls.  The
        permutation is drawn eagerly (same generator call as the eager path) into a fixed buffer; the schedule values and the Adam bias
        correction of this call's steps travel to the device in one asynchronous stream-ordered copy before the replay."""
        if self.world_size > 1:
            raise L.DwbcError("cuda_graphs=True does not capture the multi-GPU all-reduce: use world_size == 1")
        s, hp = self.storage, self._fill_hp()
        self._set_precision()
        self._packed = False
        if indices is None:
            indices, _ = s.draw_indices(self.num_mini_batches, self.generator)
        indices = indices.to(torch.int64).contiguous()
        mbs = indices.numel() // self.num_mini_batches
        self._workspace(mbs)
        if kind == "ppo":
            self._zh_buffer()
            self._diag_buffer()
        n_steps = self.num_learning_epochs * self.num_mini_batches
        key = self.graph_key(kind) + (indices.numel(),)
        g = self._graphs.get(kind)
        if g is None or g["key"] != key:
            g = self._capture(kind, key, mbs, indices.numel(), n_steps)
        g["idx"].copy_(indices)
        opt = self.optimizer if kind == "ppo" else self.hist_encoder_optimizer
        host = torch.empty(4 + 2 * n_steps, dtype=torch.float32)
        host[:3] = torch.tensor([hp.priv_reg_coef, hp.mixing_ratio, hp.torque_supervision_weight], dtype=torch.float32)
        host[3] = 0.0
        host[4:] = torch.from_numpy(L.adam_bias_correction(hp, opt.step + 1, n_steps).reshape(-1))
        g["upload"](g["scalars"], host)
        g["graph"].replay()
        opt.step += n_steps
        return hp

    def _capture(self, kind, key, mbs, n_idx, n_steps):
        self._graphs.pop(kind, None)
        scalars = torch.zeros(4 + 2 * n_steps, device=self.device)          # sched [3], pad, Adam table [n_steps, 2]
        idx = torch.zeros(n_idx, dtype=torch.int64, device=self.device)
        hp = L.PpoHyper()
        C.memmove(C.addressof(hp), C.addressof(self._hp), C.sizeof(hp))
        dev = (scalars.data_ptr(), scalars.data_ptr() + 16)
        graph = torch.cuda.CUDAGraph()
        torch.cuda.synchronize(self.device)
        with torch.cuda.graph(graph):
            if kind == "ppo":
                self._ppo_launches(hp, idx, mbs, self._ws, dev=dev)
            else:
                self._dagger_launches(hp, idx, mbs, self._ws, dev=dev)
        g = dict(key=key, graph=graph, scalars=scalars, idx=idx, hp=hp, upload=HostUpload())
        self._graphs[kind] = g
        return g

    def enforce_min_std(self):
        if self.min_policy_std is None:
            return
        ac = self.actor_critic
        self._packed = False
        L.check(self._lib.dwbc_enforce_min_std(L.ptr(ac.flat), ac.offsets["std"], L.ptr(self.min_policy_std),
                                               self.min_policy_std.numel(), L.stream_ptr()), "dwbc_enforce_min_std")

    # ------------------------------------------------------------------ checkpoint of the training state
    def _rng(self):
        """The generator `act` and `draw_indices` draw from: `generator`, or the device's default generator when it is None."""
        if self.generator is not None:
            return self.generator
        if self.device.type == "cuda":
            return torch.cuda.default_generators[self.device.index if self.device.index is not None else torch.cuda.current_device()]
        return torch.default_generator

    def _storage_shape(self):
        s = self.storage
        return None if s is None else (s.num_envs, s.num_transitions_per_env, tuple(s.obs_shape), tuple(s.actions_shape))

    def state_dict(self):
        """Everything later iterations depend on: parameters (reference names), both Adam states, `counter` (the schedules) and the
        generator state.  Precision and hyper-parameters are constructor choices and are not saved.  Taken between iterations only:
        a rollout in progress (storage.step != 0) raises DwbcError."""
        if self.storage is not None and self.storage.step != 0:
            raise L.DwbcError(f"state_dict() between iterations only: the storage holds {self.storage.step} steps of a rollout")
        sd = dict(version=CHECKPOINT_VERSION, actor_critic=self.actor_critic.state_dict(), optimizer=self.optimizer.state_dict(),
                  hist_encoder_optimizer=self.hist_encoder_optimizer.state_dict(), counter=self.counter,
                  generator=self._rng().get_state(), storage=self._storage_shape())
        if self.track_episodes:
            # the episode tracker (track_episodes > 0 only, so that checkpoints without it keep the keys of format version 1)
            sd["episodes"] = None if self._episodes is None else {k: v.clone() for k, v in self._episodes.items()}
        return sd

    def load_state_dict(self, sd):
        """Restore a state_dict() in place, so that the next iteration computes what it computed after the save.  Everything is
        checked first (format version, parameter names and shapes, storage shape, both optimizer states, generator state); a refused
        load raises DwbcError and changes nothing.  No tensor is re-bound, so captured graphs stay valid."""
        keys = {"version", "actor_critic", "optimizer", "hist_encoder_optimizer", "counter", "generator", "storage"}
        if isinstance(sd, dict) and "episodes" in sd and not self.track_episodes:
            raise L.DwbcError("the checkpoint holds an episode tracker: load it into FusedPPO(track_episodes=C > 0)")
        if self.track_episodes:
            if not isinstance(sd, dict) or "episodes" not in sd:
                raise L.DwbcError(f"this FusedPPO tracks episodes (track_episodes={self.track_episodes}): the checkpoint holds no tracker")
            keys.add("episodes")
        if not isinstance(sd, dict) or sd.get("version") != CHECKPOINT_VERSION or set(sd) != keys:
            raise L.DwbcError(f"not a FusedPPO checkpoint of format version {CHECKPOINT_VERSION}: "
                              f"version {sd.get('version') if isinstance(sd, dict) else None}")
        ac, params = self.actor_critic, sd["actor_critic"]
        if set(params) != set(ac.views):
            raise L.DwbcError(f"the checkpoint's network has other parameters: missing {[n for n in ac.views if n not in params]}, "
                              f"unexpected {[n for n in params if n not in ac.views]}")
        for n, shape in ac.manifest:
            if tuple(params[n].shape) != shape:
                raise L.DwbcError(f"parameter {n} has shape {tuple(params[n].shape)} in the checkpoint, {shape} in this network")
        if sd["storage"] != self._storage_shape():
            raise L.DwbcError(f"the checkpoint was taken with storage (envs, steps, obs, actions) {sd['storage']}, this one is "
                              f"{self._storage_shape()}")
        self.optimizer.check_state_dict(sd["optimizer"], "optimizer")
        self.hist_encoder_optimizer.check_state_dict(sd["hist_encoder_optimizer"], "hist_encoder_optimizer")
        rng, gen = self._rng(), sd["generator"]
        cur = rng.get_state()
        if not isinstance(gen, torch.Tensor) or gen.dtype != cur.dtype or gen.shape != cur.shape:
            raise L.DwbcError(f"the checkpoint's generator state does not fit the {rng.device} generator of this algorithm")
        if not isinstance(sd["counter"], int) or sd["counter"] < 0:
            raise L.DwbcError(f"counter {sd['counter']!r} is not an iteration count")
        if self.track_episodes:
            self._check_episodes(sd["episodes"])
        ac.load_state_dict(params)
        for opt, key in ((self.optimizer, "optimizer"), (self.hist_encoder_optimizer, "hist_encoder_optimizer")):
            opt.m.zero_()
            opt.v.zero_()
            opt.step = 0
            opt.load_state_dict(sd[key])
        self.counter = sd["counter"]
        rng.set_state(gen)
        if self._episodes is not None:
            for k, v in self._episodes.items():
                v.copy_(sd["episodes"][k])
        if self.storage is not None:
            self.storage.clear()             # the checkpoint was taken between iterations
        self.params_changed()

    def _check_episodes(self, ep):
        """Raise DwbcError unless `ep` is the tracker of a FusedPPO with this one's env count and track_episodes."""
        mine = self._episodes_shape()
        try:
            theirs = None if ep is None else (ep["running"].shape[0], ep["ring"].shape[0])
            if theirs != mine:
                raise L.DwbcError(f"the checkpoint's episode tracker is for (envs, capacity) {theirs}, this one for {mine}")
            if ep is not None and (set(ep) != set(self._episodes) or any(ep[k].shape != v.shape or ep[k].dtype != v.dtype
                                                                         for k, v in self._episodes.items())):
                raise L.DwbcError("the checkpoint's episode tracker is not running [N, 3] fp32, ring [C, 3] fp32, pos [2] int64")
        except (KeyError, IndexError, TypeError, AttributeError) as e:
            raise L.DwbcError(f"not an episode tracker ({type(e).__name__}: {e})") from None
