"""rl_replicas_b200 -- H100-native (sm_90a) policy-gradient update engine behind rl_replicas' Python API.

The directory is named after the reference repository (``reinforcement-learning-replications_b200``), which is not
an importable identifier; import it as ``rl_replicas_b200`` (the repo-root shim ``rl_replicas_b200.py`` maps the
name onto this directory).
"""
import logging

logging.getLogger(__name__).addHandler(logging.NullHandler())

__version__ = "0.1.0"
