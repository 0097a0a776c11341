"""Keys and default values of rl_x/algorithms/fasttd3/pytorch/default_config.py (the plugin surface: `--algorithm.<key>=...` flags and checkpoints
address them by name), except `bf16_mixed_precision_training` (False: this build is the fp32 path; True raises NotImplementedError) and
`compile_mode` (accepted, ignored).  `device` must stay "gpu": there is no CPU fallback."""
from rl_x_b200.config_dict import config_from_defaults

_DEFAULTS = (
    ('device', "gpu"),
    ('compile_mode', "reduce-overhead"),
    ('bf16_mixed_precision_training', False),
    ('total_timesteps', 2000158720),
    ('learning_rate', 3e-4),
    ('anneal_learning_rate', False),
    ('weight_decay', 0.1),
    ('batch_size', 32768),
    ('buffer_size_per_env', 10240),
    ('learning_starts', 10),  # times nr_envs
    ('v_min', -10.0),
    ('v_max', 10.0),
    ('tau', 0.1),
    ('gamma', 0.97),
    ('nr_atoms', 101),
    ('n_steps', 1),
    ('noise_std_min', 0.001),
    ('noise_std_max', 0.4),
    ('smoothing_epsilon', 0.001),
    ('smoothing_clip_value', 0.5),
    ('nr_critic_updates_per_policy_update', 2),
    ('nr_policy_updates_per_step', 1),
    ('clipped_double_q_learning', True),
    ('max_grad_norm', -1.0),  # -1.0 to disable
    ('action_clipping_and_rescaling', False),
    ('enable_observation_normalization', True),
    ('logging_frequency', 40960),
    ('evaluation_frequency', -1),
    ('save_frequency', 4096000),  # -1 to disable
    ('gemm_engine', "auto"),      # not a reference key: auto (the library's setting; exact-fp32 SIMT unless changed) | simt | tcgen05 (historical name of the 3xTF32 wgmma tensor-core engine)
)


def get_config(algorithm_name):
    return config_from_defaults(algorithm_name, _DEFAULTS)
