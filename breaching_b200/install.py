"""Mount the engine behind ``breaching.attacks.prepare_attack`` without editing the callers.

Every reference entry point (``simulate_breach.py:38``, ``benchmark_breaches.py:33``, ``minimal_example.py:48`` and
all notebooks) does ``import breaching`` and then calls ``breaching.attacks.prepare_attack(...)``.  ``install()``
rebinds that attribute on the already-importable reference package, so those scripts run unchanged; see
INTEGRATION.md for the ``sitecustomize`` one-liner.
"""
import importlib

_ORIGINAL = None


def reference_prepare_attack():
    """The reference's own ``prepare_attack`` if the original package is importable, else ``None``."""
    global _ORIGINAL
    if _ORIGINAL is not None:
        return _ORIGINAL
    try:
        ref_attacks = importlib.import_module("breaching.attacks")
    except Exception:  # noqa: BLE001 - package absent or its optional dependencies missing
        return None
    fn = getattr(ref_attacks, "prepare_attack", None)
    if fn is not None and getattr(fn, "__module__", "").startswith("breaching_b200"):
        return None
    _ORIGINAL = fn
    return fn


def install():
    """Rebind ``breaching.attacks.prepare_attack`` to the engine.  Returns the original function."""
    from . import attacks as ours

    ref_attacks = importlib.import_module("breaching.attacks")
    original = reference_prepare_attack()
    ref_attacks.prepare_attack = ours.prepare_attack
    return original


def uninstall():
    if _ORIGINAL is not None:
        importlib.import_module("breaching.attacks").prepare_attack = _ORIGINAL
