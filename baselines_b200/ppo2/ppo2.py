"""PPO2 update loop -- same keyword-only signature, defaults, schedules, logging keys and return value as the
reference's baselines/ppo2/ppo2.py:21-218 learn(), so `baselines.run` / tests can call it unchanged
(`get_learn_function('ppo2')`, run.py:154-167).

What differs is where the work happens: the rollout stays in HBM (runner.run_device), the minibatch gather of
ppo2.py:165 is an index list consumed by the kernels, and each model.train is one fused device step.  The
minibatch permutation is still drawn on the host with np.random.shuffle (ppo2.py:160, MT19937) so that a run
with the same seed visits the same minibatches as the reference; only the 8-byte indices cross PCIe.
"""
import os
import os.path as osp
import time
from collections import deque

import numpy as np
import torch

from .. import logger
from ..ops import shuffle_indices as ops_shuffle
from ..common.misc_util import constfn, explained_variance, safemean, set_global_seeds
from ..common.policies import build_policy
from .runner import Runner


def learn(*, network, env, total_timesteps, eval_env=None, seed=None, nsteps=2048, ent_coef=0.0, lr=3e-4,
          vf_coef=0.5, max_grad_norm=0.5, gamma=0.99, lam=0.95, log_interval=10, nminibatches=4, noptepochs=4,
          cliprange=0.2, save_interval=0, load_path=None, model_fn=None, update_fn=None, init_fn=None,
          mpi_rank_weight=1, comm=None, **network_kwargs):
    set_global_seeds(seed)                                                  # ppo2.py:80

    if isinstance(lr, float): lr = constfn(lr)
    else: assert callable(lr)
    if isinstance(cliprange, float): cliprange = constfn(cliprange)
    else: assert callable(cliprange)
    total_timesteps = int(total_timesteps)

    policy = build_policy(env, network, **network_kwargs)                   # ppo2.py:88
    nenvs = env.num_envs
    ob_space, ac_space = env.observation_space, env.action_space
    nbatch = nenvs * nsteps                                                 # ppo2.py:98-99
    nbatch_train = nbatch // nminibatches

    if model_fn is None:
        from .model import Model
        model_fn = Model
    model = model_fn(policy=policy, ob_space=ob_space, ac_space=ac_space, nbatch_act=nenvs,
                     nbatch_train=nbatch_train, nsteps=nsteps, ent_coef=ent_coef, vf_coef=vf_coef,
                     max_grad_norm=max_grad_norm, comm=comm, mpi_rank_weight=mpi_rank_weight)
    if not all(hasattr(model, a) for a in ("train_rollout", "step_device", "value_device", "net", "device")):
        # the rollout buffer lives in HBM and is consumed through device entry points; an object that only offers the
        # host-side step / value / train of the reference Model cannot be driven by this loop
        raise TypeError("model_fn must return a baselines_b200.ppo2 Model (or subclass, e.g. MicrobatchedModel): "
                        "got {} without the device entry points train_rollout / step_device / value_device"
                        .format(type(model).__name__))
    is_root = getattr(getattr(model, "dist", None), "rank", 0) == 0
    if load_path is not None:
        model.load(load_path)

    runner = Runner(env=env, model=model, nsteps=nsteps, gamma=gamma, lam=lam)
    eval_runner = Runner(env=eval_env, model=model, nsteps=nsteps, gamma=gamma, lam=lam) if eval_env is not None else None
    epinfobuf = deque(maxlen=100)
    eval_epinfobuf = deque(maxlen=100) if eval_env is not None else None
    if init_fn is not None:
        init_fn()

    device = model.device
    tfirststart = time.perf_counter()
    nupdates = total_timesteps // nbatch
    for update in range(1, nupdates + 1):
        assert nbatch % nminibatches == 0
        tstart = time.perf_counter()
        frac = 1.0 - (update - 1.0) / nupdates
        lrnow = lr(frac)
        cliprangenow = cliprange(frac)
        if update % log_interval == 0 and is_root: logger.info('Stepping environment...')

        ro, epinfos = runner.run_device()                                   # ppo2.py:142
        if eval_runner is not None:
            _, eval_epinfos = eval_runner.run_device()
            eval_epinfobuf.extend(eval_epinfos)
        if update % log_interval == 0 and is_root: logger.info('Done.')
        epinfobuf.extend(epinfos)

        mblossvals = run_epochs(model, ro, lrnow, cliprangenow, nbatch, nbatch_train, noptepochs, device)
        lossvals = torch.stack(mblossvals).mean(dim=0).cpu().numpy()        # one device->host sync per update
        tnow = time.perf_counter()
        fps = int(nbatch / (tnow - tstart))                                 # ppo2.py:187

        if update_fn is not None:
            update_fn(update)

        if update % log_interval == 0 or update == 1:
            values = ro.to_reference_numpy("values")
            returns = ro.to_reference_numpy("returns")
            ev = explained_variance(values, returns)
            logger.logkv("misc/serial_timesteps", update * nsteps)
            logger.logkv("misc/nupdates", update)
            logger.logkv("misc/total_timesteps", update * nbatch)
            logger.logkv("fps", fps)
            logger.logkv("misc/explained_variance", float(ev))
            logger.logkv('eprewmean', safemean([epinfo['r'] for epinfo in epinfobuf]))
            logger.logkv('eplenmean', safemean([epinfo['l'] for epinfo in epinfobuf]))
            if eval_env is not None:
                logger.logkv('eval_eprewmean', safemean([epinfo['r'] for epinfo in eval_epinfobuf]))
                logger.logkv('eval_eplenmean', safemean([epinfo['l'] for epinfo in eval_epinfobuf]))
            logger.logkv('misc/time_elapsed', tnow - tfirststart)
            for (lossval, lossname) in zip(lossvals, model.loss_names):
                logger.logkv('loss/' + lossname, float(lossval))
            if is_root:
                logger.dumpkvs()
            else:
                logger.getkvs().clear()
        if save_interval and (update % save_interval == 0 or update == 1) and logger.get_dir() and is_root:
            checkdir = osp.join(logger.get_dir(), 'checkpoints')
            os.makedirs(checkdir, exist_ok=True)
            savepath = osp.join(checkdir, '%.5i' % update)
            print('Saving to', savepath)
            model.save(savepath)
    return model


def run_epochs(model, ro, lrnow, cliprangenow, nbatch, nbatch_train, noptepochs, device, perms=None, shuffle=None):
    """The minibatch loop of ppo2.py:157-166 over a device-resident rollout.  Returns a list of device float64[5]
    loss statistics, one per minibatch.  Where the per-epoch permutation comes from:
      perms          injected permutations (parity tests);
      shuffle="host" np.random.shuffle like the reference (ppo2.py:160, MT19937): a run with the same seed visits the
                     same minibatches as the reference; the 8-byte indices cross PCIe (default, $B200RL_SHUFFLE);
      shuffle="device" a keyed bijection evaluated by a kernel (ops.shuffle_indices): nothing is generated or uploaded
                     on the host -- at cfg-3 sizes (8.4 M samples x 10 epochs) the host shuffle alone costs ~1 s per
                     update.  The key is drawn from the seeded numpy stream, so runs stay reproducible.
                     Feed-forward policies only: a recurrent one always shuffles on the host.
    Recurrent policies (ppo2.py:167-180): the permutation is over environments (perms: [noptepochs][nenvs]); a
    minibatch is nenvs / nminibatches whole environments with their rollout-start states."""
    if getattr(model, "recurrent", False):
        return _run_epochs_recurrent(model, ro, lrnow, cliprangenow, nbatch // nbatch_train, noptepochs, perms)
    out = []
    shuffle = shuffle or os.environ.get("B200RL_SHUFFLE", "host")
    inds = np.arange(nbatch) if (perms is not None or shuffle == "host") else None
    obs, actions = ro.flat("obs"), ro.flat("actions")
    returns, values, neglogp = ro.flat("returns"), ro.flat("values"), ro.flat("neglogpacs")
    for ep in range(noptepochs):
        if perms is None and shuffle == "device":
            src = ro.shuffle_buffer()
            ops_shuffle(src, nbatch, int(np.random.randint(0, 2 ** 31 - 1)) | (int(np.random.randint(0, 2 ** 31 - 1)) << 32),
                        ro.T, ro.N)
        else:
            if perms is None:
                np.random.shuffle(inds)                                      # ppo2.py:160
            else:
                inds = np.asarray(perms[ep])
            src = ro.src_index(torch.from_numpy(inds).to(device, non_blocking=True))
        for start in range(0, nbatch, nbatch_train):
            mb = src[start:start + nbatch_train]
            out.append(model.train_rollout(lrnow, cliprangenow, obs, actions, returns, values, neglogp, mb))
    return out


def _run_epochs_recurrent(model, ro, lrnow, cliprangenow, nminibatches, noptepochs, perms):
    nenvs, T = ro.N, ro.T
    assert nenvs % nminibatches == 0                                        # ppo2.py:168
    envsperbatch = nenvs // nminibatches
    envinds = np.arange(nenvs)
    flatinds = np.arange(T)[None, :] * nenvs + envinds[:, None]             # [env, t] -> buffer offset t*N + env
    obs, actions = ro.flat("obs"), ro.flat("actions")
    returns, values, neglogp = ro.flat("returns"), ro.flat("values"), ro.flat("neglogpacs")
    dones = ro.flat("dones")
    out = []
    for ep in range(noptepochs):
        if perms is None:
            np.random.shuffle(envinds)                                      # ppo2.py:172
        else:
            envinds = np.asarray(perms[ep])
        for start in range(0, nenvs, envsperbatch):
            mbenvinds = envinds[start:start + envsperbatch]                 # ppo2.py:174-176
            out.append(model.train_rollout_seq(lrnow, cliprangenow, obs, actions, returns, values, neglogp, dones,
                                               ro.states0, flatinds[mbenvinds], mbenvinds))
    return out
