from .strategy import Strategy
from .vaal import VAALQuery


class VAALSampler(VAALQuery, Strategy):
    """Drop-in for the query of active_learning/src/query_strategies/vaal_sampler.py (K9 + K1b).  Training the VAE and
    the discriminator is outside this package: pass the trained modules as vae= and discriminator=."""
