"""Keys and default values of rl_x/algorithms/ppo_lstm/flax/default_config.py.  `lstm_obs_combine_method` is "concat" or "film" and
`share_lstm_obs_encoder` either value, as in the reference (policy.py:51-59, 99-125).  `device` must stay "gpu"."""
from rl_x_b200.config_dict import config_from_defaults

_DEFAULTS = (
    ('device', "gpu"),
    ('total_timesteps', 1e9),
    ('learning_rate', 3e-4),
    ('anneal_learning_rate', False),
    ('nr_steps', 64),
    ('nr_epochs', 10),
    ('minibatch_size', 64),
    ('gamma', 0.99),
    ('gae_lambda', 0.95),
    ('clip_range', 0.2),
    ('entropy_coef', 0.0),
    ('critic_coef', 0.5),
    ('max_grad_norm', 0.5),
    ('std_dev', 1.0),
    ('obs_encoding_dim', 128),
    ('lstm_hidden_dim', 64),
    ('lstm_obs_combine_method', "concat"),
    ('share_lstm_obs_encoder', False),
    ('action_clipping_and_rescaling', True),
    ('nr_hidden_units', 256),
    ('evaluation_frequency', -1),
    ('evaluation_episodes', 10),
    ('gemm_engine', "auto"),    # not a reference key: auto (the library's setting; exact-fp32 SIMT unless changed) | simt | tcgen05 (historical name of the 3xTF32 wgmma tensor-core engine)
    ('use_cuda_graph', False),  # not a reference key: replay each minibatch update as one captured CUDA graph (same kernels, same order)
)


def get_config(algorithm_name):
    return config_from_defaults(algorithm_name, _DEFAULTS)
