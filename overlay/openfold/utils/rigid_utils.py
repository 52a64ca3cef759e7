"""Drop-in for openfold/utils/rigid_utils.py: re-exports the H100-native implementation."""
from dynamicpdb_b200.rigid_utils import *  # noqa: F401,F403
from dynamicpdb_b200.rigid_utils import (  # noqa: F401
    rot_matmul, rot_vec_mul, identity_rot_mats, identity_trans, identity_quats, quat_to_rot, rot_to_quat,
    quat_multiply, quat_multiply_by_vec, invert_rot_mat, invert_quat, Rotation, Rigid)
