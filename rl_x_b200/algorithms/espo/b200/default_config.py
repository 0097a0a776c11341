"""Same keys and defaults as rl_x/algorithms/espo/pytorch/default_config.py:4-30; `bf16_mixed_precision_training` defaults to
    False (fp32 parity path), `compile_mode` is accepted and ignored, keys specific to this build appended."""
from rl_x_b200.config_dict import config_from_defaults

_DEFAULTS = (
    ('device', "gpu"),  # a CUDA device is mandatory: there is no CPU fallback
    ('compile_mode', "reduce-overhead"),
    ('bf16_mixed_precision_training', False),
    ('total_timesteps', 1e9),
    ('learning_rate', 3e-4),
    ('anneal_learning_rate', False),
    ('nr_steps', 2048),
    ('max_epochs', 300),
    ('minibatch_size', 64),
    ('gamma', 0.99),
    ('gae_lambda', 0.95),
    ('max_ratio_delta', 0.25),
    ('delta_calc_operator', "mean"),  # mean (accumulated inside the loss kernel) | median (torch.median's lower median, radix-select kernel)
    ('entropy_coef', 0.0),
    ('critic_coef', 0.5),
    ('max_grad_norm', 0.5),
    ('std_dev', 1.0),
    ('action_clipping_and_rescaling', True),
    ('nr_hidden_units', 256),
    ('evaluation_frequency', -1),
    ('evaluation_episodes', 10),
    ('gemm_engine', "auto"),  # auto | simt (fp32 FFMA) | tcgen05 (historical name of the 3xTF32 wgmma tensor-core engine)
    ('rollout_noise', "philox"),  # philox (in-kernel counter-based normals) | torch (torch.randn on device, injected)
)


def get_config(algorithm_name):
    return config_from_defaults(algorithm_name, _DEFAULTS)
