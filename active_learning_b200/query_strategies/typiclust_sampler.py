from .strategy import Strategy
from .typiclust import TypiClustQuery


class TypiClustSampler(TypiClustQuery, Strategy):
    """TypiClust (Hacohen, Dekel & Weinshall, ICML 2022) over CoreSet's pool (K5, K15, K16, K17)."""
