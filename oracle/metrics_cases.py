"""Synthetic inputs of the metric fixture (tests/golden/metrics.pt), rebuilt from numpy's legacy seeded stream so that the
fixture stores only the reference's outputs and a checksum of the inputs.  Ground truth is fp64 (as the loader returns
atom37_pos / atom37_mask); predictions are fp32 (as the model returns them) -- tests also run them upcast to fp64."""
import numpy as np
import torch


def _unit(q):
    return q / np.linalg.norm(q, axis=-1, keepdims=True)


def _rotmats(rs, n):
    q = _unit(rs.randn(n, 4))
    w, x, y, z = q.T
    return np.stack([np.stack([w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                     np.stack([2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x)], -1),
                     np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z], -1)], -2)


def rigids(nf, N, seed):
    """gt [nf, N, 7] fp64 and pred [nf, N, 7] fp32.  Residue classes of the prediction: perturbed (most), sign-flipped
    (q vs -q), near-identical (dot ~ 1, relative perturbation 1e-9), exactly identical, and non-unit (scaled by 1.7)."""
    rs = np.random.RandomState(seed)
    q = _unit(rs.randn(nf, N, 4))
    t = 10.0 * rs.randn(nf, N, 3) + 50.0
    qp = _unit(q + 0.05 * rs.randn(nf, N, 4))
    cls = np.arange(N) % 5
    qp[:, cls == 1] *= -1.0
    qp[:, cls == 2] = q[:, cls == 2] + 1e-9 * rs.randn(nf, int((cls == 2).sum()), 4)
    qp[:, cls == 3] = q[:, cls == 3]
    qp[:, cls == 4] *= 1.7
    tp = t + rs.randn(nf, N, 3)
    gt = torch.from_numpy(np.concatenate([q, t], -1))
    pred = torch.from_numpy(np.concatenate([qp, tp], -1)).float()
    return gt, pred


def atoms(nf, N, seed, mask_kind="per_frame"):
    """gt atom37 [nf, N, 37, 3] fp64, pred [nf, N, 37, 3] fp32, mask [nf, N, 37] fp64.  The structure is a random walk of
    3.8 A steps with atoms scattered around each residue; every frame of the prediction is the truth rigidly moved
    (so superposition matters) plus 0.8 A noise.  mask_kind: "per_frame" (atoms present with p = 0.7, CA always unless
    the whole residue is empty; frames differ in their empty residues, so the mask counts differ between frames),
    "empty_frame" (the same, frame 1 entirely empty), "loader" (one [N, 37] mask shared by every frame, as the loader
    expands it)."""
    rs = np.random.RandomState(seed)
    centre = np.cumsum(3.8 * _unit(rs.randn(N, 3)), 0) + 20.0
    base = centre[:, None, :] + 1.5 * rs.randn(N, 37, 3)
    gt = base[None] + 0.5 * rs.randn(nf, N, 37, 3)
    R = _rotmats(rs, nf)
    pred = np.einsum("fij,fnaj->fnai", R, gt) + 5.0 * rs.randn(nf, 1, 1, 3) + 0.8 * rs.randn(nf, N, 37, 3)
    present = (rs.rand(N, 37) < 0.7).astype(np.float64)
    present[:, 1] = 1.0
    if mask_kind == "loader":
        present[rs.rand(N) < 0.1] = 0.0
        mask = np.broadcast_to(present, (nf, N, 37)).copy()
    else:
        mask = np.repeat(present[None], nf, 0)
        for f in range(nf):
            mask[f, rs.rand(N) < 0.1 + 0.05 * (f % 8)] = 0.0
        if mask_kind == "empty_frame":
            mask[1] = 0.0
    return torch.from_numpy(gt), torch.from_numpy(pred).float(), torch.from_numpy(mask)


def point_sets(kind, seed):
    """(reference [P, 3], coords [P, 3]) fp64 for the superposition cases: "random" (P = 130, a rotated, translated and
    noised copy), "reflected" (a mirror image: the determinant fix decides), "collinear", "coplanar", "one", "two"."""
    rs = np.random.RandomState(seed)
    R = _rotmats(rs, 1)[0]
    tr = np.array([12.0, -7.0, 30.0])
    if kind == "random":
        ref = 10.0 * rs.randn(130, 3) + 100.0
        x = (ref - 100.0) @ R.T + tr + 0.3 * rs.randn(130, 3)
    elif kind == "reflected":
        ref = 10.0 * rs.randn(60, 3)
        x = (ref * np.array([1.0, 1.0, -1.0])) @ R.T + tr + 0.1 * rs.randn(60, 3)
    elif kind == "collinear":
        s = rs.randn(20, 1) * 5.0
        ref = s * np.array([[1.0, 2.0, 2.0]]) / 3.0 + 4.0
        x = (s * np.array([[0.0, 0.6, 0.8]]) + 0.05 * rs.randn(20, 1)) @ R.T + tr
    elif kind == "coplanar":
        uv = rs.randn(25, 2) * 4.0
        ref = np.concatenate([uv, np.zeros((25, 1))], 1)
        x = ref @ R.T + tr + 0.2 * np.concatenate([rs.randn(25, 2), np.zeros((25, 1))], 1)
    elif kind == "one":
        ref, x = rs.randn(1, 3) * 10.0, rs.randn(1, 3) * 10.0
    elif kind == "two":
        ref, x = rs.randn(2, 3) * 10.0, rs.randn(2, 3) * 10.0
    else:
        raise KeyError(kind)
    return torch.from_numpy(ref), torch.from_numpy(x)


def checksum(*ts):
    """Sum of |x| and the first / last element of each tensor, fp64: the fixture stores it to prove the inputs rebuilt."""
    return torch.tensor([v for t in ts for v in (float(t.double().abs().sum()), float(t.reshape(-1)[0]), float(t.reshape(-1)[-1]))],
                        dtype=torch.float64)


# name: (builder, args) -- the fixture's cases
RIGID_CASES = {"rt_130": (3, 130, 11), "rt_1": (3, 1, 12), "rt_2": (4, 2, 13)}
ATOM_CASES = {"atoms_24": (3, 24, 21, "per_frame"), "atoms_empty_frame": (3, 24, 22, "empty_frame"),
              "atoms_2": (2, 2, 23, "per_frame")}
KABSCH_CASES = {k: 31 + i for i, k in enumerate(["random", "reflected", "collinear", "coplanar", "one", "two"])}
EVAL_WINDOW = (5, 256, 41)      # frame_time: 5 (the eval config), N = 256


def eval_window():
    """One evaluation window: rigids_0 [5, 256, 7] fp64, rigid_pred fp32, atom37_pos fp64, prot_traj[0] fp32, the loader's
    expanded mask fp64."""
    nf, N, seed = EVAL_WINDOW
    g_r, p_r = rigids(nf, N, seed)
    g_a, p_a, m = atoms(nf, N, seed + 1, "loader")
    m[:, -1, :] = 0.0
    m[:, -1, [0, 1, 2, 36]] = 1.0          # the C-terminal residue's backbone and OXT, the atom eval_fn drops
    return {"rigids_0": g_r, "rigid_pred": p_r, "atom37_pos": g_a, "atom37_pred": p_a, "atom37_mask": m}
