"""Drop-in for the reference's src/model/Dfold_network_dynamic.py: re-exports the H100-native implementation."""
from dynamicpdb_b200.Dfold_network_dynamic import *  # noqa: F401,F403
from dynamicpdb_b200.Dfold_network_dynamic import (  # noqa: F401
    FullScoreNetwork, DFOLDv2_Embeder, atom14_to_atom37, get_timestep_embedding)
