"""centertrack_b200: H100-native (sm_90a) implementation of CenterTrack's per-frame inference hot
path (DLA-34 + DCNv2 neck + heads + heat-map decode) behind the reference's Python surface."""
__version__ = '0.1.0'
