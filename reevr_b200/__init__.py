"""reevr_b200 — H100-native partitioned-convolution engine behind the FFTConvolver /
TwoStageFFTConvolver surface of tiagolr/reevr (see DESIGN.md, include/b200conv.h)."""
from .convolver import B200ConvError, Engine, FFTConvolver, Group, StereoConvolver, TwoStageFFTConvolver  # noqa: F401

__all__ = ["Engine", "Group", "FFTConvolver", "TwoStageFFTConvolver", "StereoConvolver", "B200ConvError"]
