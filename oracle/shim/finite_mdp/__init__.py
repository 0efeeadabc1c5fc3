"""Minimal stand-in for the `finite_mdp` package, which the reference's `finite_mdp()` imports to wrap its arrays
(envs/common/finite_mdp.py:92-97).  Only `finite_mdp.mdp.DeterministicMDP` is provided, and it only stores its
arguments, so `env.unwrapped.to_finite_mdp()` of the unmodified reference runs for fixture generation."""
