"""tapnet_b200: H100-native TAPIR / BootsTAPIR point-tracking inference engine.

Drop-in for the `tapnet/torch/tapir_model.py` surface of google-deepmind/tapnet:

    from tapnet_b200 import tapir_model
    model = tapir_model.TAPIR(pyramid_level=1)   # or tapir_model.build_model(path)
    model.load_state_dict(torch.load('bootstapir_checkpoint_v2.pt'))
    model = model.to('cuda').eval()
    out = model(video, query_points)
"""
from tapnet_b200.tapir_model import (FeatureGrids, QueryFeatures, TAPIR,  # noqa: F401
                                     build_model)
