"""Nexmark workload for the Z-set hot path: seeded column-major generator and
the queries the metric names (q0 plumbing, q3, q4, q7)."""
from .generator import BASE_TIME, NexmarkGenerator, STATES, state_code  # noqa: F401
from .queries import NexmarkTables, q0, q1, q2, q3, q4, q5_hop, q6, q7, q18, QUERIES  # noqa: F401
