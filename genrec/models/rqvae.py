from genrec_b200.rqvae import (MLP, Quantize, QuantizeDistance, QuantizeForwardMode, QuantizeOutput, RqVae,  # noqa: F401
                               RqVaeComputedLosses, RqVaeOutput)
