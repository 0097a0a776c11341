from rl_x_b200.plugin_properties import algorithm_properties

GeneralProperties = algorithm_properties(
    'ref: rl_x/algorithms/fasttd3/pytorch/general_properties.py (device-resident TORCH-interface environments only).',
    observations=("FLAT_VALUES",), actions=("CONTINUOUS",), interfaces=('TORCH',))
