"""breaching_b200 -- H100 (sm_90a) engine behind the breaching ``prepare_attack`` / ``reconstruct`` API."""
from .config import get_attack_config, AttackConfig  # noqa: F401

__version__ = "0.1.0"
