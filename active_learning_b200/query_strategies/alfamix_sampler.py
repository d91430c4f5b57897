from .alfamix import ALFAMixQuery
from .strategy import Strategy


class ALFAMixSampler(ALFAMixQuery, Strategy):
    """ALFA-Mix (Parvaneh et al., CVPR 2022) over CoreSet's pool (K16, K20, K5, K15, K21)."""
