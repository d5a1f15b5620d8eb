"""H100-native (sm_90a) hot path of Kaixhin/imitation-learning behind the reference's Python surface.

Importing the package does not need a GPU; creating a handle (any compute call) does — there is no CPU fallback.
"""
from . import _lib
from ._lib import build, launch_count
from .memory import ReplayMemory, TransitionBatch
from .models import (GAILDiscriminator, GMMILDiscriminator, PWILDiscriminator, REDDiscriminator, RewardRelabeller, SoftActor, TwinCritic, create_target_network, make_gail_input, manual_seed,
                     mix_expert_agent_transitions, update_target_network)
from .net import ReplicaRNG
from .optim import Adam, AdamW
from .training import adversarial_imitation_update, behavioural_cloning_update, sac_update, target_estimation_update

__all__ = ['build', 'launch_count', 'ReplayMemory', 'TransitionBatch', 'GAILDiscriminator', 'GMMILDiscriminator', 'PWILDiscriminator', 'REDDiscriminator', 'RewardRelabeller', 'SoftActor', 'TwinCritic',
           'create_target_network', 'make_gail_input', 'manual_seed', 'mix_expert_agent_transitions', 'update_target_network', 'ReplicaRNG', 'Adam', 'AdamW',
           'adversarial_imitation_update', 'behavioural_cloning_update', 'sac_update', 'target_estimation_update']
