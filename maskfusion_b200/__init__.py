"""maskfusion_b200 -- H100-native (sm_90a) implementation of MaskFusion's per-frame dense
pipeline behind the reference's MaskFusion::processFrame / Model::{performTracking,fuse,...}
interface.  The product is the CUDA library (csrc/ -> libmaskfusion_b200.so, C ABI in
include/maskfusion_b200.h); this package is the thin host-side mirror used by tests/bench."""
from .api import (MaskFusion, Model, Config, KlgLogReader, ImageLogReader, MFError, default_config, load_library, write_klg, LIB_PATH, EXPORTS, Backbone,
                  RegionProposals, roi_align, Detector, load_mask_rcnn, read_mrcnn_layer)

__all__ = ["MaskFusion", "Model", "Config", "KlgLogReader", "ImageLogReader", "MFError", "default_config", "load_library", "write_klg", "LIB_PATH", "EXPORTS", "Backbone",
           "RegionProposals", "roi_align", "Detector", "load_mask_rcnn", "read_mrcnn_layer"]
