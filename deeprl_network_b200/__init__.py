"""H100-native hot path of cts198859/deeprl_network: vectorised CACC env + A2C rollout/returns +
NeurComm/CommNet/DIAL/IA2C LSTM policies, forward and backward, as hand-written sm_90a kernels
behind the reference's IA2C/MA2C agent API.  See DESIGN.md."""
__version__ = '0.1.0'
