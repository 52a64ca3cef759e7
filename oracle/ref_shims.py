"""Import shims that let the UNMODIFIED reference (a checkout at $DFOLD_REFERENCE_ROOT) be imported here.

TEST INFRASTRUCTURE ONLY.  Nothing in the product path (dynamicpdb_b200/) may import this file.
It is used by oracle/make_golden.py (fixture generation) and by the CPU tests that pin the oracle
restatement against the live reference when that checkout is present.

The reference imports five packages at module-import time that are not installed here
(SURVEY.md §8c): tree (openfold/np/residue_constants.py:24), deepspeed
(openfold/model/primitives.py:21, openfold/utils/checkpointing.py:15), Bio
(openfold/np/protein.py:24), ml_collections (openfold/utils/loss.py:18), omegaconf
(src/data/utils.py:7,15).  None of them is used by the score-network arithmetic.
"""
import importlib.machinery
import os
import sys
import types

REFERENCE_ROOT = os.environ.get("DFOLD_REFERENCE_ROOT", "")


def reference_available() -> bool:
    return os.path.isdir(os.path.join(REFERENCE_ROOT, "src", "model"))


def _stub(name, **attrs):
    if name in sys.modules:
        return sys.modules[name]
    m = types.ModuleType(name)
    m.__spec__ = importlib.machinery.ModuleSpec(name, loader=None)
    m.__path__ = []  # behave like a package so "import a.b" works
    for k, v in attrs.items():
        setattr(m, k, v)
    sys.modules[name] = m
    return m


def _map_structure(fn, *structs):
    s0 = structs[0]
    if isinstance(s0, dict):
        return {k: _map_structure(fn, *[s[k] for s in structs]) for k in s0}
    if isinstance(s0, (list, tuple)):
        out = [_map_structure(fn, *xs) for xs in zip(*structs)]
        return type(s0)(out) if not hasattr(s0, "_fields") else type(s0)(*out)
    return fn(*structs)


class _Anything:
    """Inert attribute sink for Bio / ml_collections / omegaconf names touched at import time."""

    def __init__(self, *a, **k):
        pass

    def __call__(self, *a, **k):
        return _Anything()

    def __getattr__(self, name):
        return _Anything()


def _lenient_getattr(name):
    if name.startswith("__") and name.endswith("__"):
        raise AttributeError(name)
    return _Anything()


def install():
    """Install the stubs and put the reference on sys.path (after whatever is already there)."""
    import torch  # noqa: F401  (must be fully imported before inert stubs exist: torch inspects sys.modules)
    try:
        import tree  # noqa: F401
    except Exception:
        _stub("tree", map_structure=_map_structure)
    try:
        import deepspeed  # noqa: F401
    except Exception:
        ds = _stub("deepspeed")
        ds.utils = _stub("deepspeed.utils", is_initialized=lambda: False)
        ds.checkpointing = _stub("deepspeed.checkpointing", is_configured=lambda: False,
                                 checkpoint=lambda fn, *a: fn(*a))
        ds.comm = _stub("deepspeed.comm", is_initialized=lambda: False)
    for pkg, subs in {
        "Bio": ["Bio.PDB", "Bio.PDB.Chain", "Bio.PDB.PDBParser", "Bio.PDB.Polypeptide", "Bio.Data",
                "Bio.Data.SCOPData", "Bio.SVDSuperimposer"],
        "ml_collections": [],
        "omegaconf": [],
    }.items():
        try:
            __import__(pkg)
            continue
        except Exception:
            pass
        root = _stub(pkg)
        root.__getattr__ = _lenient_getattr  # type: ignore[attr-defined]
        for s in subs:
            m = _stub(s)
            m.__getattr__ = _lenient_getattr  # type: ignore[attr-defined]
    if reference_available() and REFERENCE_ROOT not in sys.path:
        sys.path.append(REFERENCE_ROOT)


_TRAINER_STUBS = [
    "GPUtil", "hydra", "hydra.core", "hydra.core.hydra_config", "matplotlib", "matplotlib.pyplot", "matplotlib.ticker",
    "MDAnalysis", "MDAnalysis.analysis", "MDAnalysis.analysis.rms", "MDAnalysis.analysis.align", "MDAnalysis.analysis.rdf",
    "MDAnalysis.analysis.contacts", "mdtraj", "tmtools", "pdbfixer", "simtk", "simtk.openmm", "simtk.openmm.app",
    "simtk.openmm.app.internal", "simtk.openmm.app.internal.pdbstructure", "simtk.unit", "openmm", "openmm.app", "openmm.unit",
    "openmm.app.internal", "openmm.app.internal.pdbstructure",
]


def install_trainer_stubs():
    """Inert stubs for what the reference's SCRIPTS import on top of the model (train_DFOLD_dynamics.py:17-66: GPUtil,
    hydra, matplotlib, MDAnalysis, mdtraj, the relax / openmm chain) so that `import train_DFOLD_dynamics` works here and
    the unmodified Experiment.loss_fn / inference_fn can be called on synthetic batches.  hydra.main becomes the
    identity decorator (the script decorates its `run(conf)` with it at import time, :1572)."""
    install()
    for name in _TRAINER_STUBS:
        try:
            __import__(name)
            continue
        except Exception:
            pass
        parts = name.split(".")
        for i in range(1, len(parts) + 1):
            n = ".".join(parts[:i])
            if n not in sys.modules:
                m = _stub(n)
                m.__getattr__ = _lenient_getattr  # type: ignore[attr-defined]
    import hydra
    if not callable(getattr(hydra, "main", None)) or isinstance(hydra.main, _Anything):
        hydra.main = lambda *a, **k: (lambda f: f)


def reference_experiment(model, diffuser, model_conf, exp_conf, diff_conf):
    """An `Experiment` instance of the UNMODIFIED reference trainer with just the attributes loss_fn / inference_fn read,
    built without running its constructor (which needs hydra configs, data loaders and a GPU census)."""
    install_trainer_stubs()
    import train_DFOLD_dynamics as T
    exp = object.__new__(T.Experiment)
    exp._model, exp._diffuser = model, diffuser
    exp._model_conf, exp._exp_conf, exp._diff_conf = model_conf, exp_conf, diff_conf
    return exp


def purge_reference_modules():
    """Drop cached `src.*` / `openfold.*` modules so a different overlay order can be imported."""
    for k in list(sys.modules):
        if k == "src" or k.startswith("src.") or k == "openfold" or k.startswith("openfold."):
            del sys.modules[k]
