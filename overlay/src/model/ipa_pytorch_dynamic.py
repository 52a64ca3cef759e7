"""Drop-in for the reference's src/model/ipa_pytorch_dynamic.py: re-exports the H100-native implementation."""
from dynamicpdb_b200.ipa_pytorch_dynamic import *  # noqa: F401,F403
from dynamicpdb_b200.ipa_pytorch_dynamic import (  # noqa: F401
    Linear, StructureModuleTransition, EdgeTransition, InvariantPointAttention, TorsionAngles, ScoreLayer,
    BackboneUpdate, TimeBlock, PositionalEncoding, ConvNet, MyLayerNorm, DFOLDIpaScore, AngleResnet, Rigid,
    permute_final_dims, flatten_final_dims, ipa_point_weights_init_, trunc_normal_init_, lecun_normal_init_,
    he_normal_init_, glorot_uniform_init_, final_init_, gating_init_, normal_init_, _calculate_fan)
