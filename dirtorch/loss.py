"""dirtorch.loss: the reference's training losses (APLoss, TAPLoss, their _dist variants, the triplet losses), with
the AP losses on CUDA kernels; see dirb200.loss for the differences from the reference."""
from dirb200.loss import (APLoss, APLoss_dist, TAPLoss, TAPLoss_dist, TripletLogExpLoss,  # noqa: F401
                          TripletMarginLoss, sim_to_dist)
