"""experiment/config.py: parameters and agent construction, with environments from baselines_b200.envs.make."""
import numpy as np

from ... import envs, logger
from ..ddpg import DDPG
from ..her_sampler import make_sample_her_transitions

DEFAULT_ENV_PARAMS = {
    'FetchReach-v1': {
        'n_cycles': 10,
    },
}

DEFAULT_PARAMS = {
    # env
    'max_u': 1.,  # max absolute value of actions on different coordinates
    # ddpg
    'layers': 3,  # number of layers in the critic/actor networks
    'hidden': 256,  # number of neurons in each hidden layers
    'network_class': 'baselines.her.actor_critic:ActorCritic',
    'Q_lr': 0.001,  # critic learning rate
    'pi_lr': 0.001,  # actor learning rate
    'buffer_size': int(1E6),  # for experience replay
    'polyak': 0.95,  # polyak averaging coefficient
    'action_l2': 1.0,  # quadratic penalty on actions (before rescaling by max_u)
    'clip_obs': 200.,
    'scope': 'ddpg',  # can be tweaked for testing
    'relative_goals': False,
    # training
    'n_cycles': 50,  # per epoch
    'rollout_batch_size': 2,  # per mpi thread
    'n_batches': 40,  # training batches per cycle
    'batch_size': 256,  # per mpi thread, measured in transitions and reduced to even multiple of chunk_length.
    'n_test_rollouts': 10,  # number of test rollouts per epoch, each consists of rollout_batch_size rollouts
    'test_with_polyak': False,  # run test episodes with the target network
    # exploration
    'random_eps': 0.3,  # percentage of time a random action is taken
    'noise_eps': 0.2,  # std of gaussian noise added to not-completely-random actions as a percentage of max_u
    # HER
    'replay_strategy': 'future',  # supported modes: future, none
    'replay_k': 4,  # number of additional goals used for replay, only used if off_policy_data=future
    # normalization
    'norm_eps': 0.01,  # epsilon used for observation normalization
    'norm_clip': 5,  # normalized observations are cropped to this values

    'bc_loss': 0,  # whether or not to use the behavior cloning loss as an auxilliary loss
    'q_filter': 0,  # whether or not a Q value filter should be used on the Actor outputs
    'num_demo': 100,  # number of expert demo episodes
    'demo_batch_size': 128,  # number of samples to be used from the demonstrations buffer, per mpi thread
    'prm_loss_weight': 0.001,  # Weight corresponding to the primary loss
    'aux_loss_weight': 0.0078,  # Weight corresponding to the auxilliary loss also called the cloning loss
}

# the only network class: her/actor_critic.py's, under the reference's name or this package's
NETWORK_CLASSES = ('baselines.her.actor_critic:ActorCritic', 'baselines_b200.her.actor_critic:ActorCritic')

CACHED_ENVS = {}


def cached_make_env(make_env):
    """One environment per make_env, to read the properties of the task."""
    if make_env not in CACHED_ENVS:
        CACHED_ENVS[make_env] = make_env()
    return CACHED_ENVS[make_env]


def prepare_params(kwargs):
    ddpg_params = dict()
    env_name = kwargs['env_name']

    def make_env(subrank=None):
        return envs.make(env_name)

    kwargs['make_env'] = make_env
    tmp_env = cached_make_env(kwargs['make_env'])
    assert hasattr(tmp_env, '_max_episode_steps')
    kwargs['T'] = tmp_env._max_episode_steps
    kwargs['max_u'] = np.array(kwargs['max_u']) if isinstance(kwargs['max_u'], list) else kwargs['max_u']
    kwargs['gamma'] = 1. - 1. / kwargs['T']
    if 'lr' in kwargs:
        kwargs['pi_lr'] = kwargs['lr']
        kwargs['Q_lr'] = kwargs['lr']
        del kwargs['lr']
    for name in ['buffer_size', 'hidden', 'layers', 'network_class', 'polyak', 'batch_size', 'Q_lr', 'pi_lr',
                 'norm_eps', 'norm_clip', 'max_u', 'action_l2', 'clip_obs', 'scope', 'relative_goals']:
        ddpg_params[name] = kwargs[name]
        kwargs['_' + name] = kwargs[name]
        del kwargs[name]
    kwargs['ddpg_params'] = ddpg_params
    return kwargs


def log_params(params, logger=logger):
    for key in sorted(params.keys()):
        logger.info('{}: {}'.format(key, params[key]))


# goal pairs the device reward rule is checked on: random pairs in several scales, equal goals, and pairs exactly at
# the threshold distance along each axis
def _probe_pairs(dimg, threshold):
    rng = np.random.RandomState(1234)
    a = [rng.uniform(-2, 2, (64, dimg)), rng.uniform(-1e-3, 1e-3, (16, dimg)) + 0.5, np.zeros((4, dimg))]
    b = [rng.uniform(-2, 2, (64, dimg)), np.full((16, dimg), 0.5), np.zeros((4, dimg))]
    for k in range(dimg):
        e = np.zeros((2, dimg))
        e[0, k], e[1, k] = threshold, -threshold
        a.append(np.full((2, dimg), 0.25) + e)
        b.append(np.full((2, dimg), 0.25))
    near = rng.uniform(-1, 1, (32, dimg))
    near *= threshold / np.linalg.norm(near, axis=-1, keepdims=True)
    a.append(near)
    b.append(np.zeros((32, dimg)))
    return np.concatenate(a), np.concatenate(b)


def device_reward_rule(env, dimg, info=None):
    """(reward_type, distance_threshold) when env.compute_reward is the goal-distance rule csrc/her.cu restates, bit for
    bit on a fixed probe set; None otherwise (the reward then runs on the host)."""
    u = getattr(env, 'unwrapped', env)
    rtype, thr = getattr(u, 'reward_type', None), getattr(u, 'distance_threshold', None)
    if rtype not in ('sparse', 'dense') or thr is None:
        return None
    thr = float(thr)
    a, b = _probe_pairs(dimg, thr)
    d = np.linalg.norm(a - b, axis=-1)
    want = -(d > thr).astype(np.float32) if rtype == 'sparse' else -d
    try:
        got = np.asarray(env.compute_reward(a, b, info if info is not None else {}))
    except Exception:                     # noqa: BLE001 -- a reward that cannot take the probe runs on the host
        return None
    if got.shape != want.shape or not np.array_equal(np.asarray(got, np.float32).view(np.uint32),
                                                     np.asarray(want, np.float32).view(np.uint32)):
        return None
    return rtype, thr


def configure_her(params):
    env = cached_make_env(params['make_env'])
    env.reset()

    def reward_fun(ag_2, g, info):  # vectorized
        return env.compute_reward(achieved_goal=ag_2, desired_goal=g, info=info)

    her_params = {'reward_fun': reward_fun}
    for name in ['replay_strategy', 'replay_k']:
        her_params[name] = params[name]
        params['_' + name] = her_params[name]
        del params[name]
    sample_her_transitions = make_sample_her_transitions(**her_params)
    dimg = env.observation_space.spaces['desired_goal'].shape[0]
    sample_her_transitions.device_reward = device_reward_rule(env, dimg)
    return sample_her_transitions


def simple_goal_subtract(a, b):
    assert a.shape == b.shape
    return a - b


def configure_ddpg(dims, params, reuse=False, use_mpi=True, clip_return=True):
    if params['ddpg_params']['network_class'] not in NETWORK_CLASSES:
        raise NotImplementedError(f"network_class {params['ddpg_params']['network_class']!r}: only "
                                  f"{NETWORK_CLASSES[0]} is implemented")
    sample_her_transitions = configure_her(params)
    gamma = params['gamma']
    rollout_batch_size = params['rollout_batch_size']
    ddpg_params = params['ddpg_params']
    input_dims = dims.copy()
    env = cached_make_env(params['make_env'])
    env.reset()
    ddpg_params.update({'input_dims': input_dims,
                        'T': params['T'],
                        'clip_pos_returns': True,
                        'clip_return': (1. / (1. - gamma)) if clip_return else np.inf,
                        'rollout_batch_size': rollout_batch_size,
                        'subtract_goals': simple_goal_subtract,
                        'sample_transitions': sample_her_transitions,
                        'gamma': gamma,
                        'bc_loss': params['bc_loss'],
                        'q_filter': params['q_filter'],
                        'num_demo': params['num_demo'],
                        'demo_batch_size': params['demo_batch_size'],
                        'prm_loss_weight': params['prm_loss_weight'],
                        'aux_loss_weight': params['aux_loss_weight'],
                        })
    ddpg_params['info'] = {'env_name': params['env_name']}
    for k in ('seed', 'act_cap'):
        if k in params:
            ddpg_params[k] = params[k]
    policy = DDPG(reuse=reuse, **ddpg_params, use_mpi=use_mpi)
    return policy


def configure_dims(params):
    env = cached_make_env(params['make_env'])
    env.reset()
    obs, _, _, info = env.step(env.action_space.sample())
    dims = {
        'o': obs['observation'].shape[0],
        'u': env.action_space.shape[0],
        'g': obs['desired_goal'].shape[0],
    }
    for key, value in info.items():
        value = np.array(value)
        if value.ndim == 0:
            value = value.reshape(1)
        dims['info_{}'.format(key)] = value.shape[0]
    return dims
