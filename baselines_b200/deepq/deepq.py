"""deepq.learn on the H100 kernels -- same signature, schedules, bookkeeping and return type as the reference's
baselines/deepq/deepq.py:95-332 (learn) and :23-92 (ActWrapper / load_act).

The act -> env.step -> replay.add -> sample -> train -> update_priorities -> update_target loop (deepq.py:259-307) is
unchanged; what moved to the GPU is everything inside: the replay storage and its fp64 sum / min trees live in HBM,
sampling + importance weights + the observation gather + the double-Q / Huber / clip / Adam step are device kernels,
and only the chosen action (8 bytes) and the running max priority cross PCIe per step.
"""
import os
import tempfile

import numpy as np

from .. import logger
from ..common.misc_util import set_global_seeds
from ..common.schedules import LinearSchedule
from .build_graph import DQNModel, build_act
from .replay_buffer import PrioritizedReplayBuffer, ReplayBuffer


class ActWrapper(object):
    def __init__(self, act, act_params, model=None):
        self._act = act
        self._act_params = act_params
        self.model = model
        self.initial_state = None

    def __call__(self, *args, **kwargs):
        return self._act(*args, **kwargs)

    def step(self, observation, **kwargs):
        kwargs.pop('S', None)                      # DQN has no recurrent state (deepq.py:52-54)
        kwargs.pop('M', None)
        return self._act([observation], **kwargs), None, None, None

    def save(self, path):
        """tf_util.save_variables contract: joblib dict {tf variable name: ndarray} (online + target nets)."""
        import joblib
        d = dict(self.model.q.store.export_tf("params"))
        d.update(self.model.qt.store.export_tf("params"))
        # the optimiser slots are global variables too (tf_util.py:345-355 saves all of them): a resumed run
        # continues Adam instead of restarting it
        opt = self.model.opt
        for k, v in self.model.q.store.export_tf("m").items():
            d[k.replace(":0", "/Adam:0")] = v
        for k, v in self.model.q.store.export_tf("v").items():
            d[k.replace(":0", "/Adam_1:0")] = v
        d["beta1_power:0"] = np.float32(opt.beta1 ** (opt.t + 1))
        d["beta2_power:0"] = np.float32(opt.beta2 ** (opt.t + 1))
        d["b200rl/adam_t"] = np.int64(opt.t)
        if self.model.pn is not None:                 # the noise scale / threshold and the perturbed copies are variables too
            d.update(self.model.pn.export_tf())
        dirname = os.path.dirname(path)
        if dirname:
            os.makedirs(dirname, exist_ok=True)
        joblib.dump(d, path)

    def load(self, path):
        import joblib
        d = joblib.load(os.path.expanduser(path))
        from ..ppo2.model import _adam_step_from_checkpoint
        q = self.model.q.store
        q.import_tf(d, "params")
        self.model.qt.store.import_tf(d, "params")
        q.import_tf({k.replace("/Adam:0", ":0"): v for k, v in d.items() if k.endswith("/Adam:0")}, "m")
        q.import_tf({k.replace("/Adam_1:0", ":0"): v for k, v in d.items() if k.endswith("/Adam_1:0")}, "v")
        opt = self.model.opt
        opt.t = _adam_step_from_checkpoint(d, opt.beta1, opt.beta2, opt.t)
        self.model.q.refresh()
        self.model.qt.refresh()
        if self.model.pn is not None:
            self.model.pn.import_tf(d)

    def save_act(self, path=None):
        """deepq.py:55-72: pickle of (model data, act params)."""
        import cloudpickle
        if path is None:
            path = os.path.join(logger.get_dir(), "model.pkl")
        with tempfile.TemporaryDirectory() as td:
            self.save(os.path.join(td, "model"))
            with open(os.path.join(td, "model"), "rb") as f:
                model_data = f.read()
        with open(path, "wb") as f:
            cloudpickle.dump((model_data, self._act_params), f)

    @staticmethod
    def load_act(path):
        import cloudpickle
        with open(path, "rb") as f:
            model_data, act_params = cloudpickle.load(f)
        model = DQNModel(**act_params)
        aw = ActWrapper(build_act(model), act_params, model)
        with tempfile.TemporaryDirectory() as td:
            p = os.path.join(td, "model")
            with open(p, "wb") as f:
                f.write(model_data)
            aw.load(p)
        return aw


def load_act(path):
    return ActWrapper.load_act(path)


def param_noise_threshold(eps, num_actions):
    """deepq.py:274: the KL between a greedy policy and its eps-greedy version (Plappert et al. 2017, appendix C.1)."""
    return -np.log(1.0 - eps + eps / float(num_actions))


def learn(env, network, seed=None, lr=5e-4, total_timesteps=100000, buffer_size=50000, exploration_fraction=0.1,
          exploration_final_eps=0.02, train_freq=1, batch_size=32, print_freq=100, checkpoint_freq=10000,
          checkpoint_path=None, learning_starts=1000, gamma=1.0, target_network_update_freq=500,
          prioritized_replay=False, prioritized_replay_alpha=0.6, prioritized_replay_beta0=0.4,
          prioritized_replay_beta_iters=None, prioritized_replay_eps=1e-6, param_noise=False, callback=None,
          load_path=None, **network_kwargs):
    set_global_seeds(seed)                                                    # deepq.py:190
    num_actions = env.action_space.n
    act_params = dict(ob_space=env.observation_space, num_actions=num_actions, network=network, lr=lr, gamma=gamma,
                      grad_norm_clipping=10, batch_cap=max(batch_size, 1), param_noise=param_noise,
                      **network_kwargs)                                       # deepq.py:200-208
    model = DQNModel(**act_params)
    act = ActWrapper(build_act(model), act_params, model)

    if prioritized_replay:                                                    # deepq.py:218-228
        replay_buffer = PrioritizedReplayBuffer(buffer_size, alpha=prioritized_replay_alpha, device=model.device)
        if prioritized_replay_beta_iters is None:
            prioritized_replay_beta_iters = total_timesteps
        beta_schedule = LinearSchedule(prioritized_replay_beta_iters, initial_p=prioritized_replay_beta0, final_p=1.0)
    else:
        replay_buffer = ReplayBuffer(buffer_size, device=model.device)
        beta_schedule = None
    exploration = LinearSchedule(schedule_timesteps=int(exploration_fraction * total_timesteps), initial_p=1.0,
                                 final_p=exploration_final_eps)
    model.update_target()                                                     # deepq.py:236

    episode_rewards = [0.0]
    saved_mean_reward = None
    obs = env.reset()
    reset = True
    with tempfile.TemporaryDirectory() as td:
        td = checkpoint_path or td
        model_file = os.path.join(td, "model")
        model_saved = False
        if os.path.exists(model_file):
            act.load(model_file)
            logger.log('Loaded model from {}'.format(model_file))
            model_saved = True
        elif load_path is not None:
            act.load(load_path)
            logger.log('Loaded model from {}'.format(load_path))

        for t in range(total_timesteps):
            if callback is not None:
                if callback(locals(), globals()):
                    break
            kwargs = {}
            if not param_noise:
                update_eps = exploration.value(t)
            else:
                # deepq.py:268-277: no epsilon; the KL threshold that makes the perturbed policy as far from the plain
                # one as eps-greedy with eps = exploration.value(t) would be
                update_eps = 0.0
                kwargs = dict(reset=reset, update_param_noise_scale=True,
                              update_param_noise_threshold=param_noise_threshold(exploration.value(t), num_actions))
            action = act(np.array(obs)[None], update_eps=update_eps, **kwargs)[0]
            reset = False
            new_obs, rew, done, _ = env.step(action)
            replay_buffer.add(obs, action, rew, new_obs, float(done))       # deepq.py:283
            obs = new_obs
            episode_rewards[-1] += rew
            if done:
                obs = env.reset()
                episode_rewards.append(0.0)
                reset = True

            if t > learning_starts and t % train_freq == 0:                   # deepq.py:292-303
                rb = replay_buffer
                if prioritized_replay:
                    idx, w32, _ = rb.sample_device(batch_size, beta=beta_schedule.value(t))
                else:
                    idx, w32 = rb.sample_device(batch_size)
                td_errors = model.train_device(rb._obs_t, rb._obs_tp1, rb._actions, rb._rewards, rb._dones, w32, idx,
                                               batch_size)
                if prioritized_replay:
                    rb.update_priorities_device(idx, td_errors, prioritized_replay_eps)

            if t > learning_starts and t % target_network_update_freq == 0:
                model.update_target()                                         # deepq.py:305-307

            mean_100ep_reward = round(float(np.mean(episode_rewards[-101:-1])), 1) if len(episode_rewards) > 1 else 0.0
            num_episodes = len(episode_rewards)
            if done and print_freq is not None and len(episode_rewards) % print_freq == 0:
                logger.logkv("steps", t)
                logger.logkv("episodes", num_episodes)
                logger.logkv("mean 100 episode reward", mean_100ep_reward)
                logger.logkv("% time spent exploring", int(100 * exploration.value(t)))
                logger.dumpkvs()

            if (checkpoint_freq is not None and t > learning_starts and num_episodes > 100 and t % checkpoint_freq == 0):
                if saved_mean_reward is None or mean_100ep_reward > saved_mean_reward:
                    if print_freq is not None:
                        logger.log("Saving model due to mean reward increase: {} -> {}".format(
                            saved_mean_reward, mean_100ep_reward))
                    act.save(model_file)
                    model_saved = True
                    saved_mean_reward = mean_100ep_reward
        if model_saved:
            if print_freq is not None:
                logger.log("Restored model with mean reward: {}".format(saved_mean_reward))
            act.load(model_file)
    return act
