"""Keys and default values of rl_x/algorithms/fastsac/pytorch/default_config.py (the plugin surface: `--algorithm.<key>=...` flags and checkpoints
address them by name), except `bf16_mixed_precision_training` (False: this build is the fp32 path) and `compile_mode` (accepted, ignored).
`device` must stay "gpu": there is no CPU fallback."""
from rl_x_b200.config_dict import config_from_defaults

_DEFAULTS = (
    ('device', "gpu"),
    ('compile_mode', "reduce-overhead"),
    ('bf16_mixed_precision_training', False),
    ('total_timesteps', 2000158720),
    ('learning_rate', 3e-4),
    ('anneal_learning_rate', False),
    ('weight_decay', 0.001),
    ('adam_beta1', 0.9),
    ('adam_beta2', 0.95),
    ('batch_size', 8192),
    ('buffer_size_per_env', 1024),
    ('learning_starts', 10),  # times nr_envs
    ('v_min', -20.0),
    ('v_max', 20.0),
    ('tau', 0.125),
    ('gamma', 0.97),
    ('nr_atoms', 101),
    ('n_steps', 1),
    ('target_entropy', 0.0),
    ('alpha_init', 0.001),
    ('log_std_min', -5.0),
    ('log_std_max', 0.0),
    ('nr_critic_updates_per_policy_update', 4),
    ('nr_policy_updates_per_step', 2),
    ('clipped_double_q_learning', False),
    ('max_grad_norm', -1.0),  # negative: no clipping
    ('enable_observation_normalization', True),
    ('logging_frequency', 40960),
    ('evaluation_frequency', -1),
    ('save_frequency', 4096000),  # -1 to disable
    ('gemm_engine', "auto"),      # not a reference key: auto (the library's setting; exact-fp32 SIMT unless changed) | simt | tcgen05 (historical name of the 3xTF32 wgmma tensor-core engine)
)


def get_config(algorithm_name):
    return config_from_defaults(algorithm_name, _DEFAULTS)
