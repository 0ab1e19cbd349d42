from .modules import (ConfidencePointnet, GeometryTransformer, MultiheadAttention, PositionTransformer,  # noqa: F401
                      RefineTemplate, TransformerDecoderLayer, build_network, refine_modules)
from .data import (TrackBatch, TrackTargets, combine_frames, confidence_inputs, geometry_inputs, position_inputs, revert_geometry_boxes,  # noqa: F401
                   revert_position_boxes, track_targets, tracks_from_object_infos)
from . import score  # noqa: F401
