"""PPO2 learner object on the H100 kernels -- drop-in for the reference's baselines/ppo2/model.py Model.

Same constructor keywords (model.py:27-28) and the same duck-typed protocol the reference's Runner / learn /
run.py consume (SURVEY.md 8b): step, value, train, initial_state, loss_names, save, load.  Added device
entry points (`step_device`, `value_device`, `train_rollout`) let this repo's Runner / learn keep the
rollout resident in HBM instead of round-tripping numpy.
"""
import math
import os

import numpy as np
import torch

from .. import graphs, ops
from ..common.policies import RECURRENT_NETWORKS, PolicyNet
from ..nn import Seq
from ..common import dist_util


class Model(object):
    def __init__(self, *, policy, ob_space, ac_space, nbatch_act, nbatch_train, nsteps, ent_coef, vf_coef,
                 max_grad_norm, mpi_rank_weight=1, comm=None, microbatch_size=None, device=None,
                 train_chunk=None):
        if not torch.cuda.is_available():
            raise RuntimeError("baselines_b200.ppo2.Model needs a CUDA device: the learner hot path is "
                               "hand-written sm_90a CUDA and has no CPU fallback")
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.ent_coef, self.vf_coef, self.max_grad_norm = float(ent_coef), float(vf_coef), max_grad_norm
        self.nbatch_act, self.nbatch_train, self.nsteps = nbatch_act, nbatch_train, nsteps
        chunk = int(train_chunk or os.environ.get("B200RL_TRAIN_CHUNK", 131072))
        if microbatch_size is not None:                       # microbatched_model.py:5: same maths, smaller launches
            chunk = int(microbatch_size)
        self.chunk = max(1, min(chunk, max(1, nbatch_train)))
        cap = max(nbatch_act, self.chunk)
        if getattr(policy, "network", None) in RECURRENT_NETWORKS:
            cap = max(cap, nsteps)                            # a train chunk is whole environments x nsteps
        with torch.cuda.device(self.device):
            # ortho_init consumes the GLOBAL numpy stream seeded by set_global_seeds (ppo2.py:80), like the reference
            self.net = PolicyNet(policy, cap, self.device, rng=np.random)
            self.opt = _make_optimizer(self.net.store, max_grad_norm)
            self._act_a = torch.zeros(self.net.action_shape(nbatch_act), dtype=self.net.action_dtype, device=self.device)
            self._act_v = torch.zeros(nbatch_act, dtype=torch.float32, device=self.device)
            self._act_nlp = torch.zeros(nbatch_act, dtype=torch.float32, device=self.device)
        self.loss_names = ['policy_loss', 'value_loss', 'policy_entropy', 'approxkl', 'clipfrac']   # model.py:115
        self.initial_state = None
        self.recurrent = self.net.recurrent
        if self.recurrent:
            # policies.py:90-92 / models.py lstm: zeros [nenv, 2 * nlstm] (float64, like np.zeros there)
            self.initial_state = np.zeros((nbatch_act, 2 * self.net.nlstm))
            with torch.cuda.device(self.device):
                self._act_state = torch.zeros(nbatch_act, 2 * self.net.nlstm, dtype=torch.float32, device=self.device)
                self._act_mask = torch.zeros(nbatch_act, dtype=torch.uint8, device=self.device)
        self.act_model = self.train_model = self
        self._rng_seed = int(np.random.randint(0, 2 ** 31 - 1))
        self.graphs = graphs.GraphCache()
        self._stats_out = torch.zeros(5, dtype=torch.float64, device=self.device)
        self.comm = comm
        self.dist = dist_util.DataParallel(comm, mpi_rank_weight)
        self._train_calls = 0
        self.dist.sync_from_root(self.net.store)             # model.py:131 sync_from_root
        self.net.refresh()

    # ------------------------------------------------------------------------------------ act path
    def _act_seq(self, B, state, mask, advance):
        """Recurrent networks: one step of B environments from the device state [B, 2H] float32 with the device mask
        uint8 [B] (done before this step); advance: the new state is written back in place."""
        if not self.recurrent:
            return None
        if state is None or mask is None:
            raise ValueError("a recurrent policy acts with a state and a mask (S=, M=)")
        return Seq(1, B, mask, None, state, None, state if advance else None)

    def step_device(self, obs_dev, actions, values, neglogp, noise=None, persistent=False, state=None, mask=None):
        """PolicyWithValue.step (policies.py:77-96) on device tensors; obs_dev as produced by net.encode_obs.
        persistent=True: the caller passes the same buffers on every call (the Runner's rollout slots), so the launch
        sequence is captured once per slot and replayed.  Recurrent networks: state float32 [B, 2H] is advanced in
        place, mask uint8 [B] is "done before this step"."""
        B = obs_dev.shape[0]
        seq = self._act_seq(B, state, mask, True)
        if persistent and noise is None:
            key = ("act", obs_dev.data_ptr(), actions.data_ptr(), values.data_ptr(), neglogp.data_ptr(), B)
            if seq is not None:
                key += (state.data_ptr(), mask.data_ptr())
            self.graphs.run(key, lambda: self.net.act(obs_dev, B, actions, values, neglogp, seed=self._rng_seed,
                                                      seq=seq))
        else:
            self.net.act(obs_dev, B, actions, values, neglogp, noise=noise, seed=self._rng_seed, seq=seq)

    def value_device(self, obs_dev, values, persistent=False, state=None, mask=None):
        """Recurrent networks: state / mask as in step_device; the state is not advanced (policies.py:98-119)."""
        B = obs_dev.shape[0]
        seq = self._act_seq(B, state, mask, False)

        def body():
            self.net.forward(obs_dev, B, masks=seq is None, seq=seq)
            values.copy_(self.net.v_out[:B, 0] if self.net.v_out.dim() == 2 else self.net.v_out[:B])
        if persistent:
            key = ("value", obs_dev.data_ptr(), values.data_ptr(), B)
            if seq is not None:
                key += (state.data_ptr(), mask.data_ptr())
            self.graphs.run(key, body)
        else:
            body()

    def _host_state(self, B, S, M):
        """Upload the reference's S (float [B, 2H]) and M (bool [B]) for a host-side step / value call."""
        if not self.recurrent:
            return None, None
        if B > self._act_state.shape[0]:
            st = torch.zeros(B, 2 * self.net.nlstm, dtype=torch.float32, device=self.device)
            mk = torch.zeros(B, dtype=torch.uint8, device=self.device)
        else:
            st, mk = self._act_state[:B], self._act_mask[:B]
        if S is None:
            st.zero_()
        else:
            st.copy_(torch.from_numpy(np.ascontiguousarray(S, dtype=np.float32).reshape(B, -1)))
        if M is None:
            mk.zero_()
        else:
            mk.copy_(torch.from_numpy(np.asarray(M).astype(np.uint8).reshape(B)))
        return st, mk

    def step(self, observation, S=None, M=None, noise=None, **_):
        """numpy in / numpy out, like the reference: (actions, values, states, neglogpacs).  Recurrent networks take the
        state S [B, 2H] and the mask M [B] (done before this step) and return the new state as float32; the others
        return states=None."""
        with torch.cuda.device(self.device):
            x = self.net.encode_obs(np.asarray(observation))
            B = x.shape[0]
            a, v, n = self._bufs(B)
            nz = None if noise is None else torch.as_tensor(np.ascontiguousarray(noise), dtype=torch.float32).to(self.device)
            st, mk = self._host_state(B, S, M)
            self.step_device(x, a, v, n, noise=nz, state=st, mask=mk)
            out = (self.net.actions_to_numpy(a), v.cpu().numpy(), None if st is None else st.cpu().numpy(),
                   n.cpu().numpy())
            self.net.check_obs_range()
            return out

    def value(self, ob, *args, S=None, M=None, **kwargs):
        with torch.cuda.device(self.device):
            x = self.net.encode_obs(np.asarray(ob))
            B = x.shape[0]
            _, v, _ = self._bufs(B)
            st, mk = self._host_state(B, S, M)
            self.value_device(x, v, state=st, mask=mk)
            out = v.cpu().numpy()
            self.net.check_obs_range()
            return out

    def _bufs(self, B):
        if B <= self._act_v.shape[0]:
            return self._act_a[:B], self._act_v[:B], self._act_nlp[:B]
        if B > self.net.cap:
            raise ValueError(f"batch {B} exceeds the workspace capacity {self.net.cap}")
        dev = self.device
        a = torch.zeros(self.net.action_shape(B), dtype=self.net.action_dtype, device=dev)
        return a, torch.zeros(B, device=dev), torch.zeros(B, device=dev)

    # ------------------------------------------------------------------------------------ train path
    def train_rollout(self, lr, cliprange, obs, actions, returns, values, neglogpacs, src_idx):
        """One minibatch of ppo2/model.py:133-158 on device-resident rollout arrays.

        obs/actions/returns/values/neglogpacs: flat device buffers in buffer order; src_idx: int64 device
        tensor of the M buffer offsets forming this minibatch (the shuffled `mbinds` of ppo2.py:164 mapped to
        buffer order), or None for "all rows in order".  Returns a device float64[5] of the loss statistics."""
        arrays = (obs, actions, returns, values, neglogpacs)
        M = int(src_idx.numel()) if src_idx is not None else int(returns.numel())
        idx = key = None                                         # rows in order: caller-owned temporaries, run eagerly
        with torch.cuda.device(self.device):
            if src_idx is not None:
                idx = self.graphs.home("mb_idx", max(M, self.nbatch_train), (), torch.int64, self.device)[:M]
                idx.copy_(src_idx)
                key = ("train", M) + tuple(a.data_ptr() for a in arrays)
            return self._train_step(lr, cliprange, M, returns, values, idx, self._chunks(M, self.chunk, idx, *arrays),
                                    key)

    def train_rollout_seq(self, lr, cliprange, obs, actions, returns, values, neglogpacs, dones, states0, rows, envs,
                          eager=False):
        """One recurrent minibatch of ppo2/model.py:133-158 (ppo2.py:167-180): whole environments with their start
        states.  obs/actions/returns/values/neglogpacs/dones: flat device buffers; states0: float32 [*, 2H] device;
        rows: host int64 [E, T], the buffer offsets of environment e's steps; envs: host int64 [E], its rows of
        states0.  The sequence kernels take time-major rows (t*E + e), so the launch order is built here; the loss is a
        mean, so the order does not change it.  Chunks are whole environments (chunk // T of them).  Returns a device
        float64[5] of the loss statistics.  eager: the buffers are the caller's temporaries (no graph capture)."""
        rows = np.asarray(rows, dtype=np.int64)
        envs = np.asarray(envs, dtype=np.int64).reshape(-1)
        E, T = rows.shape
        M = E * T
        per = max(1, self.chunk // T)
        spans = [(e0, min(E, e0 + per)) for e0 in range(0, E, per)]
        # per chunk, the time-major row offsets of its environments, chunk after chunk
        order = np.concatenate([rows[e0:e1].T.reshape(-1) for e0, e1 in spans])
        with torch.cuda.device(self.device):
            idx = self.graphs.home("seq_idx", max(M, self.nbatch_train), (), torch.int64, self.device)[:M]
            env = self.graphs.home("seq_env", max(E, self.nbatch_train // max(T, 1), 1), (), torch.int64,
                                   self.device)[:E]
            idx.copy_(torch.from_numpy(order))
            env.copy_(torch.from_numpy(envs))
            chunks = [(obs, (e1 - e0) * T, idx[e0 * T:e1 * T], actions, returns, values, neglogpacs,
                       Seq(T, e1 - e0, dones, idx[e0 * T:e1 * T], states0, env[e0:e1], None)) for e0, e1 in spans]
            key = None if eager else ("train_seq", E, T) + tuple(
                a.data_ptr() for a in (obs, actions, returns, values, neglogpacs, dones, states0))
            return self._train_step(lr, cliprange, M, returns, values, idx, chunks, key)

    @staticmethod
    def _chunks(M, size, idx, obs, actions, returns, values, neglogpacs):
        """M samples in chunks of at most `size`, each as loss_backward's leading arguments (x, B, src_idx, actions,
        returns, values, neglogpacs) and seq (None): gathered through idx, or (idx None) the rows in order, sliced."""
        out = []
        for s in range(0, M, size):
            B = min(size, M - s)
            if idx is not None:
                out.append((obs, B, idx[s:s + B], actions, returns, values, neglogpacs, None))
            else:
                sl = slice(s, s + B)
                out.append((obs[sl], B, None, actions[sl], returns[sl], values[sl], neglogpacs[sl], None))
        return out

    def _train_step(self, lr, cliprange, M, returns, values, idx, chunks, key):
        """The update of one minibatch of M samples from its chunks (see _chunks); idx: the minibatch's buffer offsets
        into returns / values, or None for their rows in order.  key: the graph the step is captured as and
        replayed from, or None to run it eagerly.  Runs on the current device.  Returns a device float64[5] of the loss
        statistics."""
        net, store = self.net, self.net.store
        # scalars that change from call to call go to device memory first; everything after that is a fixed launch
        # sequence for a given key, captured once and replayed (graphs.py)
        ops.set_scalars(net.clip_dev, cliprange)
        self.opt.begin_step(lr)
        inv_M = 1.0 / M

        def grads():
            store.grads.zero_()
            net.stats.zero_()
            ops.adv_stats(returns, values, idx, M, net.adv_st)                             # model.py:139
            for *args, seq in chunks:
                net.loss_backward(*args, None, self.ent_coef, self.vf_coef, inv_M, seq=seq)
            net.freeze_identity()

        def update():
            self.opt.apply()                                             # model.py:107 clip -> :114 Adam
            net.refresh()
            self._stats_out.copy_(net.stats)

        if key is None:
            grads()
            self.dist.average_gradients(store)
            update()
        elif self.dist.active and os.environ.get("B200RL_GRAPH_NCCL", "0") != "1":
            self.graphs.run(key + ("grads",), grads)
            self.dist.average_gradients(store)                           # mpi_adam_optimizer.py:39-40, BEFORE the clip
            self.graphs.run(key + ("update",), update)
        else:
            # single process: one graph per minibatch.  (B200RL_GRAPH_NCCL=1 also captures the NCCL all-reduce;
            # measured on 2 GPUs it is no faster than the split form -- 236.7 vs 236.6 ms -- and the process
            # group then hangs at teardown, so the split form is the default.)
            self.graphs.run(key, lambda: (grads(), self.dist.average_gradients(store), update()),
                            allow_fallback=self.dist.active)
        self._after_train_call()
        return self._stats_out / M

    def _after_train_call(self):
        """mpi_adam_optimizer.py:41-42: every 100th compute_gradients call checks that the ranks still hold identical
        parameters (check_synced :53-68); a mismatch is a hard error there (assert) and here."""
        self._train_calls += 1
        if self.dist.active and self._train_calls % 100 == 0:
            if not self.dist.check_synced(self.net.store):
                raise AssertionError("parameters are not synchronised across ranks (check_synced, "
                                     "mpi_adam_optimizer.py:53-68) after {} train calls".format(self._train_calls))

    def train(self, lr, cliprange, obs, returns, masks, actions, values, neglogpacs, states=None):
        """Reference signature (model.py:133); numpy minibatch in, list of 5 python floats out.  Recurrent networks:
        the rows are whole environments, env-major (row e * nsteps + t, ppo2.py:174-176), and states [nenv, 2H] are
        their start states."""
        if states is not None and not self.recurrent:
            raise NotImplementedError("states are only taken by recurrent policies ('lstm', 'cnn_lstm')")
        if states is None and self.recurrent:
            raise ValueError("a recurrent policy trains from the start states of its minibatch (states=)")
        with torch.cuda.device(self.device):
            dev = self.device
            x = self.net.encode_obs(np.asarray(obs))
            a = torch.as_tensor(np.ascontiguousarray(actions), dtype=self.net.action_dtype).to(dev).contiguous()
            f = lambda z: torch.as_tensor(np.ascontiguousarray(z), dtype=torch.float32).to(dev)
            # the buffers are this call's temporaries: both kinds run eagerly (eager=True; src_idx None)
            if self.recurrent:
                T = self.nsteps
                E = int(np.shape(states)[0])
                assert x.shape[0] == E * T, "a recurrent minibatch is nenv whole sequences of nsteps"
                m = torch.from_numpy(np.asarray(masks).astype(np.uint8).reshape(-1)).to(dev)
                rows = np.arange(E * T, dtype=np.int64).reshape(E, T)
                st = self.train_rollout_seq(float(lr), float(cliprange), x, a, f(returns), f(values), f(neglogpacs),
                                            m, f(np.asarray(states).reshape(E, -1)), rows, np.arange(E),
                                            eager=True)
            else:
                st = self.train_rollout(float(lr), float(cliprange), x, a, f(returns), f(values), f(neglogpacs), None)
            out = [float(s) for s in st.cpu().numpy()]
            self.net.check_obs_range()
            return out

    # ------------------------------------------------------------------------------------ checkpoints
    def save(self, save_path):
        """tf_util.save_variables (tf_util.py:345-355): joblib dict {tf variable name: ndarray}.  Adam slots
        are stored under the TF slot names '<var>/Adam:0', '<var>/Adam_1:0' like the reference's global
        variables."""
        import joblib
        d = dict(self.net.store.export_tf("params"))
        for k, v in self.net.store.export_tf("m").items():
            d[k.replace(":0", "/Adam:0")] = v
        for k, v in self.net.store.export_tf("v").items():
            d[k.replace(":0", "/Adam_1:0")] = v
        d["beta1_power:0"] = np.float32(self.opt.beta1 ** (self.opt.t + 1))
        d["beta2_power:0"] = np.float32(self.opt.beta2 ** (self.opt.t + 1))
        # float32 beta1_power underflows to 0 after ~1000 Adam steps (62 PPO2 updates at the defaults), so the step
        # count cannot be recovered from it; it is stored explicitly under a key no TF variable uses
        d["b200rl/adam_t"] = np.int64(self.opt.t)
        if self.net.obs_rms is not None:                     # RunningMeanStd variables (mpi_running_mean_std.py:11-26)
            for k, name in self.net.rms_names.items():
                d[name] = np.array(self.net.obs_rms[k], dtype=np.float64)
        dirname = os.path.dirname(save_path)
        if dirname:
            os.makedirs(dirname, exist_ok=True)
        joblib.dump(d, save_path)

    def load(self, load_path):
        import joblib
        d = joblib.load(os.path.expanduser(load_path))
        store = self.net.store
        store.import_tf({k: v for k, v in d.items() if k in store.tf_map}, "params")
        store.import_tf({k.replace("/Adam:0", ":0"): v for k, v in d.items() if k.endswith("/Adam:0")}, "m")
        store.import_tf({k.replace("/Adam_1:0", ":0"): v for k, v in d.items() if k.endswith("/Adam_1:0")}, "v")
        self.opt.t = _adam_step_from_checkpoint(d, self.opt.beta1, self.opt.beta2, self.opt.t)
        if self.net.obs_rms is not None:
            self.net.set_obs_rms({k: d[name] for k, name in self.net.rms_names.items() if name in d})
        self.net.refresh()

    # parameters in the reference's TF naming / layout (used by the parity tests)
    def get_params(self):
        return self.net.store.export_tf("params")

    def set_params(self, params):
        self.net.store.import_tf(params, "params")
        self.net.refresh()


def _adam_step_from_checkpoint(d, beta1, beta2, default):
    """Adam step count of a checkpoint.  Our own files carry it as an integer; a reference (TF) checkpoint only has
    the float32 accumulators beta1_power = beta1^(t+1), beta2_power = beta2^(t+1) (tf.train.AdamOptimizer slots saved
    by tf_util.save_variables, tf_util.py:345-355).  beta1_power is denormal / zero after ~800 steps, so beta2_power
    (usable up to ~9e4 steps) is preferred; once both have underflowed the bias correction is 1 to fp32 precision and
    any large t gives the same update."""
    if "b200rl/adam_t" in d:
        return int(d["b200rl/adam_t"])
    tiny = float(np.finfo(np.float32).tiny)
    for key, beta in (("beta2_power:0", beta2), ("beta1_power:0", beta1)):
        if key in d:
            p = float(d[key])
            if p >= 1.0:
                return 0
            if p > tiny * 1e3:                       # well inside the normal range: log() is accurate
                return max(0, int(round(math.log(p) / math.log(beta))) - 1)
    if "beta1_power:0" in d or "beta2_power:0" in d:
        return 10 ** 6                               # both underflowed: sqrt(1-b2^t)/(1-b1^t) == 1
    return default


def _make_optimizer(store, max_grad_norm):
    from ..nn import Optimizer
    return Optimizer(store, eps=1e-5, max_grad_norm=max_grad_norm)       # model.py:100 epsilon=1e-5
