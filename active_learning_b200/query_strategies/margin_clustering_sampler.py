from .margin_clustering import MarginClusteringQuery
from .strategy import Strategy


class MarginClusteringSampler(MarginClusteringQuery, Strategy):
    """Drop-in for active_learning/src/query_strategies/margin_clustering_sampler.py (K1 + K7 + K8)."""
