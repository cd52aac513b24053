"""`stoix` import path of this build: every `stoix.<module>` resolves to `stoix_b200.<module>` (same module object),
so code written against the reference -- `from stoix.systems.ppo.anakin.ff_ppo import learner_setup`,
`from stoix.utils.multistep import batch_truncated_generalized_advantage_estimation`, Hydra `_target_: stoix.networks...`
strings -- runs on this framework unchanged.  The script-style launches of the reference
(`python stoix/systems/ppo/anakin/ff_ppo.py k=v ...`, stoix/systems/ppo/anakin/ff_ppo.py:709-727) exist as thin files
under this directory."""
import importlib
import importlib.abc
import importlib.util
import sys

_PREFIX, _REAL = "stoix.", "stoix_b200."


class _AliasFinder(importlib.abc.MetaPathFinder, importlib.abc.Loader):
    def find_spec(self, fullname, path=None, target=None):
        if not fullname.startswith(_PREFIX):
            return None
        real = _REAL + fullname[len(_PREFIX):]
        try:
            if importlib.util.find_spec(real) is None:
                return None
        except (ImportError, ValueError):
            return None
        return importlib.util.spec_from_loader(fullname, self)

    def create_module(self, spec):
        return importlib.import_module(_REAL + spec.name[len(_PREFIX):])

    def exec_module(self, module):
        return None


# FIRST on the meta path: once `stoix.networks` is the stoix_b200.networks package object, the regular path finder would
# otherwise find `torso.py` through its __path__ and execute it a second time under the alias name.
if not any(isinstance(f, _AliasFinder) for f in sys.meta_path):
    sys.meta_path.insert(0, _AliasFinder())
