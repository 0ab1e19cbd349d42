from .modules import (ConfidencePointnet, GeometryTransformer, MultiheadAttention, PositionTransformer,  # noqa: F401
                      RefineTemplate, TransformerDecoderLayer, build_network, refine_modules)
from .data import (TrackBatch, combine_frames, confidence_inputs, geometry_inputs, position_inputs, revert_geometry_boxes,  # noqa: F401
                   revert_position_boxes, tracks_from_object_infos)
