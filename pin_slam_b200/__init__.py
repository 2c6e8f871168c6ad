"""pin_slam_b200 -- H100-native (sm_90a) hot path of PIN-SLAM behind the reference's
NeuralPoints / Decoder API.  See DESIGN.md and INTEGRATION.md."""
__version__ = "0.1.0"
