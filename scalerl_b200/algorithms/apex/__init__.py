from .actor import B200ApexActor, apex_epsilons
from .learner import (APEX_DUELING_PARAM_NAMES, APEX_NOISY_DUELING_PARAM_NAMES, APEX_NOISY_PARAM_NAMES, APEX_PARAM_NAMES, ApexHParams,
                      AtariQNet, B200ApexLearner, NoisyLinear, apex_param_names, apex_param_shapes, categorical_support,
                      default_q_state_dict, quantile_taus)

__all__ = ['APEX_DUELING_PARAM_NAMES', 'APEX_NOISY_DUELING_PARAM_NAMES', 'APEX_NOISY_PARAM_NAMES', 'APEX_PARAM_NAMES', 'ApexHParams', 'AtariQNet', 'B200ApexActor', 'B200ApexLearner', 'NoisyLinear', 'apex_epsilons',
           'apex_param_names', 'apex_param_shapes', 'categorical_support', 'default_q_state_dict', 'quantile_taus']
