"""Dump the numeric residue tables the score-network epilogue reads (SURVEY.md §2 row 17:
"constants are *read* by the hot path; import as-is") into dynamicpdb_b200/data/residue_tables.npz,
so the product and the oracle run without a checkout of the reference.

Sources (reference file:line):
  src/data/residue_constants.py:778-781  restype_atom14_to_rigid_group / _mask / _rigid_group_positions,
                                          restype_rigid_group_default_frame  (used by src/data/all_atom.py:13-18)
  openfold/np/residue_constants.py:1341-1342  RESTYPE_ATOM37_TO_ATOM14, RESTYPE_ATOM37_MASK
                                          (used by src/model/Dfold_network_dynamic.py:579,587)
Run here (reference mounted):  python oracle/make_constants.py
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_shims  # noqa: E402

ref_shims.install()
from src.data import residue_constants as src_rc  # noqa: E402
from openfold.np import residue_constants as of_rc  # noqa: E402
from openfold.data.data_transforms import get_chi_atom_indices  # noqa: E402

out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                   "dynamicpdb_b200", "data", "residue_tables.npz")
np.savez_compressed(
    out,
    default_frames=np.asarray(src_rc.restype_rigid_group_default_frame, dtype=np.float32),   # [21,8,4,4]
    atom14_group=np.asarray(src_rc.restype_atom14_to_rigid_group, dtype=np.int64),           # [21,14]
    atom14_mask=np.asarray(src_rc.restype_atom14_mask, dtype=np.float32),                    # [21,14]
    atom14_pos=np.asarray(src_rc.restype_atom14_rigid_group_positions, dtype=np.float32),    # [21,14,3]
    atom37_to_atom14=np.asarray(of_rc.RESTYPE_ATOM37_TO_ATOM14, dtype=np.int64),             # [21,37]
    atom37_mask=np.asarray(of_rc.RESTYPE_ATOM37_MASK, dtype=np.float32),                     # [21,37]
    # input featurisation (openfold/data/data_transforms.py:895-919, :1001-1003, :1068-1070)
    chi_atom_indices=np.asarray(get_chi_atom_indices(), dtype=np.int64),                     # [21,4,4]
    chi_angles_mask=np.asarray(list(of_rc.chi_angles_mask) + [[0.0] * 4], dtype=np.float32), # [21,4]
    chi_pi_periodic=np.asarray(of_rc.chi_pi_periodic, dtype=np.float32),                     # [21,4]
)
# sanity: the two copies of the tables in the reference agree
assert np.array_equal(src_rc.restype_rigid_group_default_frame, of_rc.restype_rigid_group_default_frame)
print("wrote", out, os.path.getsize(out), "bytes")
