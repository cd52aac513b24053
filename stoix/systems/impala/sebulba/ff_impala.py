"""Launch file with the reference's path (`python stoix/systems/impala/sebulba/ff_impala.py k=v ...`); the implementation is
stoix_b200/systems/impala/sebulba/ff_impala.py, and `import stoix.systems.impala.sebulba.ff_impala` yields that very module."""
import os
import sys

_ROOT = os.path.abspath(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "..", "..", ".."))
if _ROOT not in sys.path:
    sys.path.insert(0, _ROOT)
from stoix_b200.systems.impala.sebulba import ff_impala as _impl  # noqa: E402

if __name__ == "__main__":
    _impl.hydra_entry_point()
else:
    sys.modules[__name__] = _impl
