"""MicrobatchedModel -- same constructor contract and the same arithmetic as baselines/ppo2/microbatched_model.py:

  * advantages are normalised over the FULL minibatch (:43),
  * every microbatch of `microbatch_size` samples yields the gradient of its own mean loss, which passes through
    the MPI mean (it is `compute_gradients` of the MpiAdamOptimizer) and through clip_by_global_norm *per microbatch*
    (:60 fetches `self.grads`, the clipped tensors of ppo2/model.py:105-107),
  * the clipped microbatch gradients are summed and divided by their number (:63-70), one Adam step applies them
    (:70-73; no second clip), and the statistics are the mean over microbatches (:75).

This differs from the plain `Model(train_chunk=...)` chunking (accumulate, then clip once), which is the arithmetic of
the reference's plain Model; the two coincide whenever no microbatch norm exceeds max_grad_norm."""
import torch

from .. import ops
from .model import Model


class MicrobatchedModel(Model):
    def __init__(self, *, policy, ob_space, ac_space, nbatch_act, nbatch_train, nsteps, ent_coef, vf_coef,
                 max_grad_norm, mpi_rank_weight=1, comm=None, microbatch_size=None, **kw):
        self.nmicrobatches = nbatch_train // microbatch_size
        self.microbatch_size = microbatch_size
        assert nbatch_train % microbatch_size == 0, \
            'microbatch_size ({}) should divide nbatch_train ({}) evenly'.format(microbatch_size, nbatch_train)
        super().__init__(policy=policy, ob_space=ob_space, ac_space=ac_space, nbatch_act=nbatch_act,
                         nbatch_train=nbatch_train, nsteps=nsteps, ent_coef=ent_coef, vf_coef=vf_coef,
                         max_grad_norm=max_grad_norm, mpi_rank_weight=mpi_rank_weight, comm=comm,
                         microbatch_size=microbatch_size, **kw)
        self._acc = torch.zeros_like(self.net.store.grads)

    def train(self, lr, cliprange, obs, returns, masks, actions, values, neglogpacs, states=None):
        assert states is None, "microbatches with recurrent models are not supported yet"    # microbatched_model.py:36
        return super().train(lr, cliprange, obs, returns, masks, actions, values, neglogpacs)

    def train_rollout_seq(self, *args, **kwargs):
        raise AssertionError("microbatches with recurrent models are not supported yet")

    def train_rollout(self, lr, cliprange, obs, actions, returns, values, neglogpacs, src_idx):
        net, store, opt = self.net, self.net.store, self.opt
        M = int(src_idx.numel()) if src_idx is not None else int(returns.numel())
        mb = self.microbatch_size
        assert M % mb == 0, "minibatch of {} samples is not a multiple of microbatch_size {}".format(M, mb)
        nmicro = M // mb
        with torch.cuda.device(self.device):
            self._acc.zero_()
            net.stats.zero_()
            ops.adv_stats(returns, values, src_idx, M, net.adv_st)        # microbatched_model.py:43: FULL minibatch
            for *args, _ in self._chunks(M, mb, src_idx, obs, actions, returns, values, neglogpacs):
                store.grads.zero_()
                net.loss_backward(*args, cliprange, self.ent_coef, self.vf_coef, 1.0 / mb)
                net.freeze_identity()
                self.dist.average_gradients(store)                        # inside compute_gradients, before the clip
                clip = opt.clip if opt.clip is not None else 0.0
                if clip > 0:
                    ops.sumsq(store.grads, opt.sumsq)
                ops.clip_accumulate(store.grads, self._acc, clip, 1.0 / nmicro, opt.sumsq if clip > 0 else None)
            store.grads.copy_(self._acc)
            opt.step(lr, clip=False)
            net.refresh()
            self._after_train_call()
            return net.stats / M
