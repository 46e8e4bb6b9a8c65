"""The plugin type.

When the reference package is importable at import time its own `polyfuzz.models.BaseMatcher` is the base
class, so this package's matchers ARE reference plugins.  Otherwise an identical ABC is defined here (mirror of
polyfuzz/models/_base.py:6-31: abstract match(), attributes model_id and type) and, should `polyfuzz`
become importable later in the process, every matcher class is registered with the reference's ABC as a
virtual subclass -- either way `isinstance(m, polyfuzz.models.BaseMatcher)` holds and
`PolyFuzz(method=TFIDF(...))` (polyfuzz/polyfuzz.py:127-151) works unmodified."""
import sys
from abc import ABC, abstractmethod
from typing import List

import pandas as pd

try:                                                    # pragma: no cover - depends on the environment
    from polyfuzz.models import BaseMatcher as _RefBaseMatcher
    BaseMatcher = _RefBaseMatcher
    REFERENCE_BASE = True
except Exception:                                       # reference not importable now: same contract, own ABC
    REFERENCE_BASE = False

    class BaseMatcher(ABC):
        """The abstract BaseMatching to be modelled after for string matching"""

        def __init__(self, model_id: str = "Model 0"):
            self.model_id = model_id
            self.type = "Base Model"
            register_with_reference(type(self))

        @abstractmethod
        def match(self, from_list: List[str], to_list: List[str] = None, **kwargs) -> pd.DataFrame:
            """Returns a DataFrame with columns From, To, Similarity (one row per from_list element)."""
            raise NotImplementedError()

_REGISTERED = set()


def register_with_reference(cls) -> bool:
    """Register `cls` as a virtual subclass of the reference's BaseMatcher if `polyfuzz` is loaded."""
    if REFERENCE_BASE or cls in _REGISTERED:
        return True
    mod = sys.modules.get("polyfuzz.models")
    ref = getattr(mod, "BaseMatcher", None) if mod is not None else None
    if ref is None:
        return False
    ref.register(cls)
    _REGISTERED.add(cls)
    return True
