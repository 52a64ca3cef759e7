"""Drop-in for openfold/model/structure_module.py: re-exports the H100-native implementation."""
from dynamicpdb_b200.structure_module import *  # noqa: F401,F403
from dynamicpdb_b200.structure_module import (  # noqa: F401
    AngleResnetBlock, AngleResnet, InvariantPointAttention, BackboneUpdate, StructureModuleTransitionLayer,
    StructureModuleTransition, StructureModule)
