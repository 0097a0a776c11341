"""Same keys and defaults as rl_x/algorithms/sac/pytorch/default_config.py:4-28 (bf16 autocast off: this is the fp32 parity path;
    compile_mode accepted and ignored)."""
from rl_x_b200.config_dict import config_from_defaults

_DEFAULTS = (
    ('device', "gpu"),
    ('compile_mode', "reduce-overhead"),
    ('bf16_mixed_precision_training', False),
    ('total_timesteps', 1e9),
    ('learning_rate', 3e-4),
    ('anneal_learning_rate', False),
    ('buffer_size', 1e6),
    ('learning_starts', 5000),
    ('batch_size', 256),
    ('tau', 0.005),
    ('gamma', 0.99),
    ('target_entropy', "auto"),
    ('log_std_min', -20),
    ('log_std_max', 2),
    ('nr_hidden_units', 256),
    ('logging_frequency', 300),
    ('evaluation_frequency', -1),
    ('evaluation_episodes', 10),
    ('use_cuda_graph', True),  # replay the whole update (noise + ~58 kernels) as one CUDA graph
    ('gemm_engine', "auto"),  # auto | simt (fp32 FFMA) | tcgen05 (historical name of the 3xTF32 wgmma tensor-core engine)
)


def get_config(algorithm_name):
    return config_from_defaults(algorithm_name, _DEFAULTS)
