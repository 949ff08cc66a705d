"""Python host-side mirror of the reference interface over the C ABI
(include/maskfusion_b200.h).  Names follow the reference: MaskFusion.processFrame,
Model.performTracking / predictIndices / fuse / clean / combinedPredict
(Core/MaskFusion.h:69-70, Core/Model/Model.h:128-164).

There is NO CPU fallback: if libmaskfusion_b200.so is missing or no CUDA device is
present, construction raises.
"""
from __future__ import annotations

import ctypes as C
import os
import re

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libmaskfusion_b200.so")
_LIB = None


class MFError(RuntimeError):
    pass


class Config(C.Structure):
    """mf_config (include/maskfusion_b200.h)"""
    _fields_ = [
        ("width", C.c_int32), ("height", C.c_int32),
        ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float),
        ("depthCutoff", C.c_float), ("maxDepthProcessed", C.c_float), ("icpWeight", C.c_float),
        ("rgbOnly", C.c_int32), ("pyramid", C.c_int32), ("fastOdom", C.c_int32), ("so3", C.c_int32),
        ("frameToFrameRGB", C.c_int32),
        ("confGlobal", C.c_float), ("confObject", C.c_float),
        ("timeDelta", C.c_int32), ("outlierCoeff", C.c_float),
        ("capacityGlobal", C.c_int32), ("capacityObject", C.c_int32),
        ("enableMultipleModels", C.c_int32), ("trackAllModels", C.c_int32), ("modelSpawnOffset", C.c_int32),
        ("minRelSizeNew", C.c_float), ("maxRelSizeNew", C.c_float),
        ("segThreshold", C.c_float), ("segWeightDistance", C.c_float), ("segWeightConvexity", C.c_float),
        ("segMorphEdgeIterations", C.c_int32), ("segMorphEdgeRadius", C.c_int32),
        ("segMorphMaskIterations", C.c_int32), ("segMorphMaskRadius", C.c_int32),
    ]


HEADER = os.path.join(HERE, "..", "include", "maskfusion_b200.h")
# ctypes type of each scalar the header uses; every pointer is c_void_p (c_char_p for strings), so no handle is truncated to int
_SCALARS = {"int": C.c_int, "unsigned": C.c_uint, "int64_t": C.c_int64, "float": C.c_float, "double": C.c_double}


def _spaced(t: str) -> str:
    return " ".join(t.replace("*", " * ").split()).replace(" *", "*")          # "const char *" -> "const char*"


def _prototypes():
    """[(name, return type, [parameter types])] of every mf_* function the header declares, types as written there ("const char*")"""
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/|//[^\n]*", " ", src, flags=re.S)         # comments
    src = re.sub(r"^\s*#[^\n]*", " ", src, flags=re.M)                 # preprocessor lines
    out = []
    for ret, name, params in re.findall(r"([^;{}()]*?)\b(mf_\w+)\s*\(([^()]*)\)\s*;", src):
        types = []
        for p in params.split(","):
            p, array = re.subn(r"\[[^\]]*\]\s*$", "", p.strip())         # float pose16[16] is a float*
            p = re.sub(r"(?<=[\s*])\w+$", "", p.strip())                 # the parameter's name
            types.append(_spaced(p) + "*" * array)
        out.append((name, _spaced(ret), [] if types == ["void"] else types))
    return out


def _ctype(decl: str, where: str):
    t = _spaced(re.sub(r"\b(const|struct)\b", "", decl))
    if t == "void":
        return None
    if t == "char*":
        return C.c_char_p
    if t.endswith("*"):
        return C.c_void_p
    if t in _SCALARS:
        return _SCALARS[t]
    raise MFError(f"{where}: no ctypes binding for the type '{decl.strip()}' ({HEADER})")


EXPORTS = tuple(name for name, _, _ in _prototypes())


def load_library():
    """dlopen the in-tree CUDA library and bind every function of include/maskfusion_b200.h; loud failure if it has not been built"""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = LIB_PATH
    tag = os.environ.get("MFB200_TAG")          # A/B builds of the same library (maskfusion_b200/build.py), e.g. another CTA shape
    if tag:
        path = LIB_PATH.replace(".so", f"_{tag}.so")
    if not os.path.exists(path):
        raise MFError(f"{path} not found: run `python -m maskfusion_b200.build` (there is no CPU fallback)")
    L = C.CDLL(path)
    for name, ret, params in _prototypes():
        if not hasattr(L, name):
            raise MFError(f"{path} lacks {name}, which the header declares: rebuild it (`python -m maskfusion_b200.build`)")
        f = getattr(L, name)
        f.restype = _ctype(ret, name)
        f.argtypes = [_ctype(p, name) for p in params]
    _LIB = L
    return L


def _error() -> MFError:
    """the message of the calling thread's last failed call (mf_last_error)"""
    return MFError(load_library().mf_last_error().decode())


def default_config(width=640, height=480, **kw) -> Config:
    c = Config()
    load_library().mf_config_defaults(C.byref(c), width, height)
    for k, v in kw.items():
        if not hasattr(c, k):
            raise AttributeError(k)
        setattr(c, k, v)
    return c


def _p(a):
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.c_void_p)


class Model:
    """Handle on one surfel model (reference: class Model, Core/Model/Model.h)."""

    def __init__(self, mf: "MaskFusion", index: int):
        self.mf, self.i = mf, index

    def _ck(self, r):
        return self.mf._ck(r)

    def getPose(self) -> np.ndarray:
        out = np.zeros(16, np.float32)
        self._ck(self.mf.L.mf_get_pose(self.mf.h, self.i, _p(out)))
        return out.reshape(4, 4).T.copy()          # column-major ABI -> numpy row-major

    def overridePose(self, T: np.ndarray):
        a = np.ascontiguousarray(np.asarray(T, np.float32).T).ravel()
        self._ck(self.mf.L.mf_set_pose(self.mf.h, self.i, _p(a)))

    def debugSetPoses(self, pose: np.ndarray, lastPose: np.ndarray):
        a = np.ascontiguousarray(np.asarray(pose, np.float32).T).ravel()
        b = np.ascontiguousarray(np.asarray(lastPose, np.float32).T).ravel()
        self._ck(self.mf.L.mf_debug_set_poses(self.mf.h, self.i, _p(a), _p(b)))

    def getClassID(self) -> int:
        return self.mf.L.mf_model_class_id(self.mf.h, self.i)

    def getID(self) -> int:
        return self.mf.L.mf_model_id(self.mf.h, self.i)

    def lastCount(self) -> int:
        return self._ck(self.mf.L.mf_model_surfel_count(self.mf.h, self.i))

    def setConfidenceThreshold(self, t: float):
        self._ck(self.mf.L.mf_model_set_conf_threshold(self.mf.h, self.i, float(t)))

    def downloadMap(self) -> np.ndarray:
        n = self.lastCount()
        out = np.zeros((max(n, 1), 12), np.float32)
        got = self._ck(self.mf.L.mf_download_surfels(self.mf.h, self.i, _p(out), n))
        return out[:got]

    def uploadMap(self, surfels: np.ndarray):
        s = np.ascontiguousarray(surfels, np.float32)
        self._ck(self.mf.L.mf_upload_surfels(self.mf.h, self.i, _p(s), s.shape[0]))

    def initialise(self, time: int):
        self._ck(self.mf.L.mf_model_init_from_frame(self.mf.h, self.i, time))

    def performTracking(self) -> np.ndarray:
        out = np.zeros(16, np.float32)
        self._ck(self.mf.L.mf_model_perform_tracking(self.mf.h, self.i, _p(out)))
        return out.reshape(4, 4).T.copy()

    def predictIndices(self, time: int):
        self._ck(self.mf.L.mf_model_predict_indices(self.mf.h, self.i, time))

    def fuse(self, time: int, depthCutoff: float, weightMultiplier: float = 1.0):
        self._ck(self.mf.L.mf_model_fuse(self.mf.h, self.i, time, depthCutoff, weightMultiplier))

    def clean(self, time: int):
        self._ck(self.mf.L.mf_model_clean(self.mf.h, self.i, time))

    def combinedPredict(self, time: int, maxTime: int):
        self._ck(self.mf.L.mf_model_combined_predict(self.mf.h, self.i, time, maxTime))

    # ---- read-back (reference layouts) ----
    def indexMap(self):
        H, W = self.mf.H, self.mf.W
        idx = np.zeros((H, W), np.uint32); vc = np.zeros((H, W, 4), np.float32)
        ct = np.zeros((H, W, 4), np.float32); nr = np.zeros((H, W, 4), np.float32)
        self._ck(self.mf.L.mf_download_index_map(self.mf.h, self.i, _p(idx), _p(vc), _p(ct), _p(nr)))
        return idx, vc, ct, nr

    def prediction(self):
        H, W = self.mf.H, self.mf.W
        im = np.zeros((H, W, 4), np.uint8); vc = np.zeros((H, W, 4), np.float32)
        nr = np.zeros((H, W, 4), np.float32); tt = np.zeros((H, W), np.uint16)
        self._ck(self.mf.L.mf_download_prediction(self.mf.h, self.i, _p(im), _p(vc), _p(nr), _p(tt)))
        return im, vc, nr, tt

    def fillIn(self):
        H, W = self.mf.H, self.mf.W
        im = np.zeros((H, W, 4), np.uint8); v = np.zeros((H, W, 4), np.float32); n = np.zeros((H, W, 4), np.float32)
        self._ck(self.mf.L.mf_download_fill_in(self.mf.h, self.i, _p(im), _p(v), _p(n)))
        return im, v, n

    def association(self):
        H, W = self.mf.H, self.mf.W
        flag = np.zeros((W, H), np.uint8); best = np.zeros((W, H), np.uint32); meas = np.zeros((W, H, 12), np.float32)
        self._ck(self.mf.L.mf_download_association(self.mf.h, self.i, _p(flag), _p(best), _p(meas)))
        return flag, best, meas

    def modelMaps(self, level: int):
        H, W = self.mf.H >> level, self.mf.W >> level
        v = np.zeros((3, H, W), np.float32); n = np.zeros((3, H, W), np.float32)
        self._ck(self.mf.L.mf_download_model_maps(self.mf.h, self.i, level, _p(v), _p(n)))
        return v, n

    def trackStats(self):
        A = np.zeros((6, 6)); b = np.zeros(6); e = np.zeros(6, np.float32)
        self._ck(self.mf.L.mf_download_track_stats(self.mf.h, self.i, _p(A), _p(b), _p(e)))
        return A, b, e

    def icpStep(self, level: int, Rcurr: np.ndarray, tcurr: np.ndarray) -> np.ndarray:
        out = np.zeros(29, np.float32)
        R = np.ascontiguousarray(Rcurr, np.float32).ravel(); t = np.ascontiguousarray(tcurr, np.float32).ravel()
        self._ck(self.mf.L.mf_icp_step(self.mf.h, self.i, level, _p(R), _p(t), _p(out)))
        return out

    def poseLog(self) -> np.ndarray:
        n = self._ck(self.mf.L.mf_pose_log_size(self.mf.h, self.i))
        out = np.zeros((max(n, 1), 8))
        got = self._ck(self.mf.L.mf_get_pose_log(self.mf.h, self.i, _p(out), n))
        return out[:got]


class MaskFusion:
    """reference: class MaskFusion (Core/MaskFusion.h).  `stream` is a raw cudaStream_t
    (int); pass torch.cuda.current_stream().cuda_stream to time with torch events."""

    def __init__(self, cfg: Config | None = None, device: int = 0, stream: int | None = None, **kw):
        self.L = load_library()
        self.cfg = cfg if cfg is not None else default_config(**kw)
        self.W, self.H = self.cfg.width, self.cfg.height
        self.h = self.L.mf_create(C.byref(self.cfg), device, C.c_void_p(stream) if stream else None)
        if not self.h:
            raise _error()

    def _ck(self, r):
        if r < 0:
            raise _error()
        return r

    def close(self):
        if getattr(self, "h", None):
            self.L.mf_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def exportPoses(self, exportDir: str) -> int:
        """MaskFusion::exportPoses: <exportDir>poses-<id>.txt per model"""
        return self._ck(self.L.mf_export_poses(self.h, exportDir.encode()))

    def processFrame(self, rgb: np.ndarray, depth: np.ndarray, timestamp: int = 0, mask=None, inPose=None,
                     weightMultiplier: float = 1.0, bootstrap: bool = False, classIDs=None):
        """bool MaskFusion::processFrame(FrameDataPointer, const Eigen::Matrix4f*, float, bool); mask/classIDs are
        FrameData::mask / FrameData::classIDs (external instance masks, Core/FrameData.h:36-40)"""
        if classIDs is not None:
            c = np.ascontiguousarray(classIDs, np.int32)
            self._ck(self.L.mf_set_frame_classes(self.h, _p(c), int(c.shape[0])))
        if mask is not None:
            if mask.dtype != np.uint8 or mask.shape != (self.H, self.W):
                raise MFError("mask must be HxW uint8 (CV_8UC1)")
            mask = np.ascontiguousarray(mask)
        if rgb.dtype != np.uint8 or rgb.shape != (self.H, self.W, 3):
            raise MFError("rgb must be HxWx3 uint8 (CV_8UC3, MaskFusion.cpp:202)")
        if depth.dtype != np.float32 or depth.shape != (self.H, self.W):
            raise MFError("depth must be HxW float32 metres (CV_32FC1, MaskFusion.cpp:201)")
        ip = None if inPose is None else np.ascontiguousarray(np.asarray(inPose, np.float32).T).ravel()
        self._ck(self.L.mf_process_frame(self.h, _p(np.ascontiguousarray(rgb)), _p(np.ascontiguousarray(depth)), int(timestamp),
                                         _p(mask), _p(ip), float(weightMultiplier), int(bootstrap)))
        return False

    def processFramePtr(self, rgb_ptr: int, depth_ptr: int, timestamp: int = 0, on_device: bool = False, mask_ptr: int = 0):
        """raw-pointer variant (pinned host or device memory), used by bench.py; class ids through setFrameClasses"""
        fn = self.L.mf_process_frame_device if on_device else self.L.mf_process_frame
        self._ck(fn(self.h, C.c_void_p(rgb_ptr), C.c_void_p(depth_ptr), int(timestamp), C.c_void_p(mask_ptr) if mask_ptr else None, None, 1.0, 0))

    def attachBackbone(self, backbone, every_k: int = 5):
        """Mask R-CNN backbone on the frame path: every k-th processFrame enqueues mold + forward on the backbone's stream"""
        self._ck(self.L.mf_attach_backbone(self.h, C.c_void_p(backbone.h) if backbone is not None else None, int(every_k)))

    def attachDetector(self, detector, every_k: int = 1):
        """Mask R-CNN detector on the frame path (mf_attach_detector): segmentation frames given no mask take the detector's id image
        and class ids every k-th tick; None detaches.  The context does not own the detector: detach before closing it."""
        self._ck(self.L.mf_attach_detector(self.h, C.c_void_p(detector.h) if detector is not None else None, int(every_k)))

    def frameMasks(self):
        """-> (mask H x W uint8, class ids) that segmentation read on the last frame (FrameData::mask / classIDs); ([all zero], [])
        when the frame carried no masks"""
        m = np.zeros((self.H, self.W), np.uint8); c = np.zeros(256, np.int32); n = C.c_int(0)
        self._ck(self.L.mf_download_frame_masks(self.h, _p(m), _p(c), C.byref(n)))
        return m, c[:n.value].tolist()

    def setFrameClasses(self, classIDs):
        c = np.ascontiguousarray(classIDs, np.int32)
        self._ck(self.L.mf_set_frame_classes(self.h, c.ctypes.data_as(C.c_void_p), int(c.shape[0])))

    def setFrame(self, rgb, depth, mask=None):
        self._ck(self.L.mf_set_frame(self.h, _p(np.ascontiguousarray(rgb)), _p(np.ascontiguousarray(depth)), _p(mask)))

    def segmentation(self):
        m = np.zeros((self.H, self.W), np.uint8); p = np.zeros((self.H, self.W), np.uint8)
        multi = bool(self.cfg.enableMultipleModels)
        self._ck(self.L.mf_download_segmentation(self.h, _p(m), _p(p) if multi else None))
        return m, p

    def sync(self):
        self._ck(self.L.mf_sync(self.h))

    def setProfiling(self, on: bool):
        self._ck(self.L.mf_set_profiling(self.h, int(on)))

    def stageTimes(self) -> dict:
        """{kernel name: (launch count, total device ms)} measured with CUDA events on the pipeline's stream"""
        buf = C.create_string_buffer(1 << 16)
        self._ck(self.L.mf_get_stage_times(self.h, buf, len(buf)))
        out = {}
        for line in buf.value.decode().splitlines():
            n, c, ms = line.split()
            out[n] = (int(c), float(ms))
        return out

    def getTick(self) -> int:
        return self.L.mf_tick(self.h)

    def setFrameQueue(self, n: int):
        """the reference's queueLength (-frameQ, mf_set_frame_queue): each processFrame pushes its frame and processes the oldest one
        once n frames are queued; 0 or 1 = no queue.  Before the first frame."""
        self._ck(self.L.mf_set_frame_queue(self.h, int(n)))

    def frameQueueSize(self) -> int:
        """frames queued and not yet processed"""
        return self._ck(self.L.mf_frame_queue_size(self.h))

    def kernelLaunches(self) -> int:
        return int(self.L.mf_kernel_launches(self.h))

    def getModels(self):
        return [Model(self, i) for i in range(self.L.mf_model_count(self.h))]

    def getBackgroundModel(self) -> Model:
        return Model(self, 0)

    def filteredDepth(self):
        out = np.zeros((self.H, self.W), np.float32)
        self._ck(self.L.mf_download_filtered_depth(self.h, _p(out)))
        return out

    def frameMaps(self, level: int):
        H, W = self.H >> level, self.W >> level
        d = np.zeros((H, W), np.float32); v = np.zeros((3, H, W), np.float32); n = np.zeros((3, H, W), np.float32)
        self._ck(self.L.mf_download_frame_maps(self.h, level, _p(d), _p(v), _p(n)))
        return d, v, n

    def edgeMap(self):
        e = np.zeros((self.H, self.W), np.float32); b = np.zeros((self.H, self.W), np.uint8)
        self._ck(self.L.mf_download_edge_map(self.h, _p(e), _p(b)))
        return e, b

    def morphClose(self, image, radius: int, iterations: int, ellipse: bool = True):
        """test hook: GPU close of a host image; ellipse=True: the mask-id close (MfSegmentation.cpp:424-426), False: the binary
        edge-map close (segmentation.cu:217-255) -> (closed, inverted)"""
        a = np.ascontiguousarray(image, np.uint8).copy()
        assert a.shape == (self.H, self.W)
        inv = np.zeros_like(a)
        self._ck(self.L.mf_morph_close(self.h, _p(a), int(radius), int(iterations), int(ellipse), None if ellipse else _p(inv)))
        return a if ellipse else (a, inv)


class KlgLogReader:
    """reference: class KlgLogReader (GUI/Tools/KlgLogReader.{h,cpp})"""

    def __init__(self, path: str, width: int, height: int, flipColors: bool = False):
        self.L = load_library()
        self.W, self.H = width, height
        self.k = self.L.mf_klg_open(path.encode(), width, height, int(flipColors))
        if not self.k:
            raise _error()

    def getNumFrames(self):
        return self.L.mf_klg_num_frames(self.k)

    def hasMore(self):
        return bool(self.L.mf_klg_has_more(self.k))

    def getNext(self):
        rgb = np.zeros((self.H, self.W, 3), np.uint8); depth = np.zeros((self.H, self.W), np.float32)
        ts = C.c_int64(0)
        if self.L.mf_klg_get_next(self.k, _p(rgb), _p(depth), C.byref(ts)) != 0:
            raise _error()
        return rgb, depth, ts.value

    def close(self):
        if self.k:
            self.L.mf_klg_close(self.k)
            self.k = None


def write_ply(path: str, surfels: np.ndarray, conf_threshold: float) -> int:
    """one model's cloud as MaskFusion::savePly writes it (MaskFusion.cpp:733-848); surfels = Model.downloadMap()"""
    L = load_library()
    a = np.ascontiguousarray(surfels, np.float32).reshape(-1, 12)
    n = L.mf_write_ply(path.encode(), _p(a) if a.size else None, int(a.shape[0]), float(conf_threshold))
    if n < 0:
        raise _error()
    return n


def generate_id_image(result: dict, min_score: float, class_filter=(), special_assignments=()):
    """reference: generate_id_image(result, min_score, class_filter, special_assignments), MaskRCNN/helpers.py:70-98.
    result = {'masks': HxWxN uint8, 'scores': N, 'class_ids': N, 'rois': Nx4} -> (id_image HxW uint8, class ids, rois)"""
    L = load_library()
    masks = np.ascontiguousarray(result["masks"], np.uint8)
    H, W, N = masks.shape
    scores = np.ascontiguousarray(result["scores"], np.float32); cls = np.ascontiguousarray(result["class_ids"], np.int32)
    rois = np.ascontiguousarray(result["rois"], np.int32).reshape(N, 4)
    cf = np.ascontiguousarray(list(class_filter), np.int32); sa = np.ascontiguousarray(list(special_assignments), np.int32)
    img = np.zeros((H, W), np.uint8); ec = np.zeros(max(N, 1), np.int32); er = np.zeros((max(N, 1), 4), np.int32)
    n = L.mf_generate_id_image(_p(masks), H, W, N, _p(scores), _p(cls), _p(rois), float(min_score), _p(cf) if cf.size else None, int(cf.size),
                               _p(sa) if sa.size else None, int(sa.size), _p(img), _p(ec), _p(er))
    if n < 0:
        raise _error()
    return img, ec[:n].tolist(), er[:n].tolist()


def pre_segmentation(mask: np.ndarray, depth: np.ndarray, model_ids, next_model_id: int, allow_new: bool, mapping: np.ndarray):
    """PreSegmentation::performSegmentation (PreSegmentation.cpp:28-90).  mapping: uint8[256], updated in place (state across frames).
    -> (fullSegmentation HxW u8, hasNewLabel, superPixelCount, depthMean, depthStd) with one entry per model (+1 with a new label)"""
    L = load_library()
    m = np.ascontiguousarray(mask, np.uint8); d = np.ascontiguousarray(depth, np.float32)
    H, W = m.shape
    ids = np.ascontiguousarray(model_ids, np.uint8)
    assert mapping.dtype == np.uint8 and mapping.size == 256 and mapping.flags["C_CONTIGUOUS"]
    seg = np.zeros((H, W), np.uint8); has_new = C.c_int(0)
    spc = np.zeros(len(ids) + 1, np.uint32); mean = np.zeros(len(ids) + 1, np.float32); std = np.zeros(len(ids) + 1, np.float32)
    n = L.mf_pre_segmentation(_p(m), _p(d), W, H, _p(ids), len(ids), int(next_model_id), int(bool(allow_new)), _p(mapping), _p(seg), C.byref(has_new),
                              _p(spc), _p(mean), _p(std))
    if n < 0:
        raise _error()
    return seg, bool(has_new.value), spc[:n].copy(), mean[:n].copy(), std[:n].copy()


def decode_exr_depth(buf: bytes) -> np.ndarray:
    """OpenEXR scan-line file -> HxW float32 depth as the -dir reader delivers it (csrc/mf_loader.cu: decodeEXRDepth)"""
    L = load_library()
    w, h = C.c_int(0), C.c_int(0)
    a = np.frombuffer(buf, np.uint8)
    if L.mf_decode_exr_depth(_p(a), int(a.shape[0]), None, 0, C.byref(w), C.byref(h)) != 0:
        raise _error()
    out = np.zeros((h.value, w.value), np.float32)
    if L.mf_decode_exr_depth(_p(a), int(a.shape[0]), _p(out), out.size, C.byref(w), C.byref(h)) != 0:
        raise _error()
    return out


def decode_jpeg(buf: bytes) -> np.ndarray:
    """baseline JPEG -> HxWx3 uint8 RGB, bit-identical to libjpeg's default decode (csrc/mf_jpeg.cu)"""
    L = load_library()
    w, h = C.c_int(0), C.c_int(0)
    a = np.frombuffer(buf, np.uint8)
    if L.mf_decode_jpeg(_p(a), int(a.shape[0]), None, 0, C.byref(w), C.byref(h)) != 0:
        raise _error()
    out = np.zeros((h.value, w.value, 3), np.uint8)
    if L.mf_decode_jpeg(_p(a), int(a.shape[0]), _p(out), out.size, C.byref(w), C.byref(h)) != 0:
        raise _error()
    return out


class ImageLogReader:
    """reference: class ImageLogReader (GUI/Tools/ImageLogReader.{h,cpp}), the "-dir" loader: colour / depth / optional mask images
    named <prefix><zero-padded index><ext> (+ "<mask>.txt" with class ids and boxes)"""

    def __init__(self, colorDirectory: str, depthDirectory: str | None = None, maskDirectory: str | None = None, indexWidth: int = 4,
                 colorPrefix: str = "", depthPrefix: str = "", maskPrefix: str = ""):
        self.L = load_library()
        enc = lambda v: v.encode() if v else None          # noqa: E731
        self.r = self.L.mf_dir_open(colorDirectory.encode(), enc(depthDirectory), enc(maskDirectory), indexWidth, colorPrefix.encode(),
                                    depthPrefix.encode(), maskPrefix.encode())
        if not self.r:
            raise _error()
        w, h = C.c_int(0), C.c_int(0)
        self.L.mf_dir_size(self.r, C.byref(w), C.byref(h))
        self.W, self.H = w.value, h.value

    def getNumFrames(self):
        return self.L.mf_dir_num_frames(self.r)

    def hasMore(self):
        return bool(self.L.mf_dir_has_more(self.r))

    def hasMasks(self):
        return bool(self.L.mf_dir_has_masks(self.r))

    def setMaxMasks(self, n: int):
        self.L.mf_dir_set_max_masks(self.r, n)

    def getNext(self):
        """-> rgb, depth, timestamp, mask or None, classIDs or None, rois (n,4 as x,y,w,h) or None   (FrameData fields)"""
        rgb = np.zeros((self.H, self.W, 3), np.uint8); depth = np.zeros((self.H, self.W), np.float32); mask = np.zeros((self.H, self.W), np.uint8)
        ids = np.zeros(256, np.int32); boxes = np.zeros((255, 4), np.int32); n = C.c_int(256); ts = C.c_int64(0)
        rc = self.L.mf_dir_get_next(self.r, _p(rgb), _p(depth), _p(mask), _p(ids), _p(boxes), C.byref(n), C.byref(ts))
        if rc < 0:
            raise _error()
        cls = ids[:n.value].copy() if n.value else None
        return rgb, depth, ts.value, (mask if rc == 1 else None), cls, (boxes[:n.value - 1].copy() if n.value > 1 else None)

    def close(self):
        if self.r:
            self.L.mf_dir_close(self.r)
            self.r = None


def write_klg(path: str, timestamps, depth_mm: np.ndarray, rgb: np.ndarray):
    """raw .klg (layout: KlgLogReader.cpp:29,53-89)"""
    L = load_library()
    n, H, W = depth_mm.shape
    ts = np.ascontiguousarray(timestamps, np.int64)
    d = np.ascontiguousarray(depth_mm, np.uint16); c = np.ascontiguousarray(rgb, np.uint8)
    if L.mf_klg_write(path.encode(), W, H, n, _p(ts), _p(d), _p(c)) != 0:
        raise _error()


class _CnnHandle:
    """what the Mask R-CNN handles share: errors through mf_last_error (a None handle is a failed create), close() through their destroy
    function"""

    _destroy = ""

    def _ck(self, r):
        if r is None or r < 0:
            raise _error()
        return r

    def close(self):
        if getattr(self, "h", None):
            getattr(self.L, self._destroy)(self.h); self.h = None


class Backbone(_CnnHandle):
    """Mask R-CNN ResNet-101-FPN backbone on wgmma GEMMs (csrc/mf_cnn.cu).  Weights are synthetic (seeded) unless loaded with
    loadWeights (matterport's Keras arrays in a safetensors file, BatchNorm folded; see load_mask_rcnn)."""

    _destroy = "mf_backbone_destroy"

    def __init__(self, input_size=1024, seed=1, stream: int | None = None):
        self.L = load_library()
        self.S = input_size
        self.h = self._ck(self.L.mf_backbone_create(input_size, seed, C.c_void_p(stream) if stream else None))

    def layers(self):
        out = []
        for i in range(self.L.mf_backbone_num_layers(self.h)):
            d = np.zeros(6, np.int32)
            self.L.mf_backbone_layer(self.h, i, _p(d))
            out.append(tuple(int(v) for v in d))
        return out

    def weights(self, i):
        cin, cout, k, stride, pad, kpad = self.layers()[i]
        w = np.zeros((cout, kpad), np.float32); b = np.zeros(cout, np.float32)
        self.L.mf_backbone_get_weights(self.h, i, _p(w), _p(b))
        return w[:, :k * k * cin].reshape(cout, k, k, cin), b

    def loadWeights(self, path: str):
        """the backbone's tensors of a safetensors weight file (conv1, res*, bn*, fpn_*); all or nothing, complete on return"""
        self._ck(self.L.mf_backbone_load_weights(self.h, os.fsencode(path)))
        return self

    def forward(self, input_ptr: int):
        self._ck(self.L.mf_backbone_forward(self.h, C.c_void_p(input_ptr)))

    def output(self, level):
        d = np.zeros(3, np.int32)
        ptr = self.L.mf_backbone_output(self.h, level, _p(d))
        return ptr, tuple(int(v) for v in d)

    def download(self, level) -> np.ndarray:
        """bf16 output as float32 numpy (H, W, C)"""
        _, (h, w, c) = self.output(level)
        raw = np.zeros((h, w, c), np.uint16)
        self._ck(self.L.mf_backbone_download(self.h, level, _p(raw)))
        return _bf16_to_f32(raw)

    def flops(self):
        return float(self.L.mf_backbone_flops(self.h))

    def numGemms(self):
        return int(self.L.mf_backbone_num_gemms(self.h))


def _bf16_to_f32(raw: np.ndarray) -> np.ndarray:
    return (raw.astype(np.uint32) << 16).view(np.float32)


class RegionProposals(_CnnHandle):
    """Mask R-CNN RPN head + proposal layer + pyramid ROI Align on a Backbone's P2..P6 (csrc/mf_rpn.cu).  Weights are synthetic (seeded)
    unless loaded with loadWeights.  Runs on the backbone's stream; close it before the backbone."""

    POST_NMS, POOL, CHANNELS = 1000, 7, 256
    CONV, HEADS, PROPOSALS, ROI_ALIGN = 1, 2, 4, 8        # stage bits of run()
    _destroy = "mf_rpn_destroy"

    def __init__(self, backbone: Backbone, seed=1):
        self.L = load_library()
        self.backbone = backbone
        self.S = backbone.S
        self.h = self._ck(self.L.mf_rpn_create(C.c_void_p(backbone.h), seed))
        self.A = int(self.L.mf_rpn_num_anchors(self.h))

    def forward(self):
        """conv, heads, proposals and ROI Align of the backbone's last forward"""
        self._ck(self.L.mf_rpn_forward(self.h))

    def run(self, stages: int):
        self._ck(self.L.mf_rpn_run(self.h, int(stages)))

    def anchors(self) -> np.ndarray:
        out = np.zeros((self.A, 4), np.float32)
        self._ck(self.L.mf_rpn_get_anchors(self.h, _p(out)))
        return out

    def headOutputs(self):
        """fp32 (logits [A, 2], deltas [A, 4])"""
        lg = np.zeros((self.A, 2), np.float32); dl = np.zeros((self.A, 4), np.float32)
        self._ck(self.L.mf_rpn_get_head_outputs(self.h, _p(lg), _p(dl)))
        return lg, dl

    def convOutput(self, level: int) -> np.ndarray:
        """shared 3x3 conv output of P(level+2), level 0..4, as float32 (H, W, 512)"""
        n = self.S >> (level + 2)
        raw = np.zeros((n, n, 512), np.uint16)
        self._ck(self.L.mf_rpn_download_conv(self.h, int(level), _p(raw)))
        return _bf16_to_f32(raw)

    def proposals(self):
        """-> (kept count, rois [1000, 4] normalised y1 x1 y2 x2, zero rows past the count)"""
        rois = np.zeros((self.POST_NMS, 4), np.float32)
        n = self._ck(self.L.mf_rpn_get_proposals(self.h, _p(rois)))
        return n, rois

    def pooled(self, raw: bool = False) -> np.ndarray:
        """ROI-aligned features [1000, 7, 7, 256]: bf16 bit patterns (uint16) if raw, else float32"""
        out = np.zeros((self.POST_NMS, self.POOL, self.POOL, self.CHANNELS), np.uint16)
        self._ck(self.L.mf_rpn_get_pooled(self.h, _p(out)))
        return out if raw else _bf16_to_f32(out)

    def weights(self):
        """-> conv weights [512, 3, 3, 256], conv bias [512], head weights [18, 512] (rows 0..5 logits a*2+c, 6..17 deltas a*4+k),
        head bias [18]; bf16-representable float32"""
        cw = np.zeros((512, 3, 3, 256), np.float32); cb = np.zeros(512, np.float32)
        hw = np.zeros((18, 512), np.float32); hb = np.zeros(18, np.float32)
        self._ck(self.L.mf_rpn_get_weights(self.h, _p(cw), _p(cb), _p(hw), _p(hb)))
        return cw, cb, hw, hb

    def loadWeights(self, path: str):
        """rpn_conv_shared, rpn_class_raw and rpn_bbox_pred of a safetensors weight file; all or nothing, complete on return"""
        self._ck(self.L.mf_rpn_load_weights(self.h, os.fsencode(path)))
        return self

    def propose(self, logits_ptr: int, deltas_ptr: int, anchors_ptr: int, n: int):
        """the proposal stage on caller-supplied device arrays (float32 [n, 2], [n, 4], [n, 4]); results through proposals()"""
        self._ck(self.L.mf_rpn_propose(self.h, C.c_void_p(logits_ptr), C.c_void_p(deltas_ptr), C.c_void_p(anchors_ptr), int(n)))


def roi_align(backbone: Backbone, boxes_ptr: int, n: int, pool: int, out_ptr: int):
    """pyramid ROI Align of n normalised boxes (device float32 [n, 4]) on the backbone's P2..P5 into out (device bf16 [n, pool, pool, 256]),
    enqueued on the backbone's stream"""
    L = load_library()
    if L.mf_roi_align_bf16(C.c_void_p(backbone.h), C.c_void_p(boxes_ptr) if n else None, int(n), int(pool), C.c_void_p(out_ptr) if n else None) != 0:
        raise _error()


class Detector(_CnnHandle):
    """Mask R-CNN detection heads on a RegionProposals' proposals (csrc/mf_heads.cu): classifier, detection layer, mask head, unmould and
    generate_id_image.  Weights are synthetic (seeded) unless loaded with loadWeights.  Runs on the backbone's stream; close it before the
    RegionProposals."""

    ROIS, MAX_DETECTIONS, NUM_CLASSES, MASK = 1000, 100, 81, 28
    CLASSIFIER, DETECTIONS, MASKS, ID_IMAGE = 1, 2, 4, 8        # stage bits of run()
    _destroy = "mf_detector_destroy"

    def __init__(self, rpn: RegionProposals, seed=1):
        self.L = load_library()
        self.rpn = rpn
        self.h = self._ck(self.L.mf_detector_create(C.c_void_p(rpn.h), seed))

    def run(self, stages: int):
        self._ck(self.L.mf_detector_run(self.h, int(stages)))

    def forward(self, image_w: int, image_h: int):
        """every head stage on the RPN's last forward, for an original image of image_w x image_h"""
        self._ck(self.L.mf_detector_forward(self.h, int(image_w), int(image_h)))

    def detect(self, rgba_ptr: int, W: int, H: int):
        """mould + backbone + RPN + heads of a W x H RGBA8 device image, enqueued on the backbone's stream"""
        self._ck(self.L.mf_detector_detect(self.h, C.c_void_p(rgba_ptr), int(W), int(H)))

    def set_export(self, min_score=0.55, class_filter=(), special_assignments=()):
        """generate_id_image's arguments for the id-image stage"""
        cf = np.ascontiguousarray(list(class_filter), np.int32); sa = np.ascontiguousarray(list(special_assignments), np.int32)
        self._ck(self.L.mf_detector_set_export(self.h, float(min_score), _p(cf) if cf.size else None, int(cf.size), _p(sa) if sa.size else None,
                                               int(sa.size)))

    def refine(self, rois_ptr: int, logits_ptr: int, deltas_ptr: int, n: int):
        """the detection layer on device arrays (float32 [n, 4], [n, 81], [n, 81, 4]); results through detections()"""
        self._ck(self.L.mf_detector_refine(self.h, C.c_void_p(rois_ptr), C.c_void_p(logits_ptr), C.c_void_p(deltas_ptr), int(n)))

    def paste(self, detections_ptr: int, masks_ptr: int, W: int, H: int):
        """unmould + id image of device arrays (float32 [100, 6], [100, 28, 28]) for a W x H image; results through idImage()"""
        self._ck(self.L.mf_detector_paste(self.h, C.c_void_p(detections_ptr), C.c_void_p(masks_ptr), int(W), int(H)))

    def layers(self):
        """(Cin, rows, k, stride, pad, K) per layer: FC1, FC2, heads, 4 mask convs, transposed conv, mask logits"""
        out = []
        for i in range(self.L.mf_detector_num_layers(self.h)):
            d = np.zeros(6, np.int32)
            self._ck(self.L.mf_detector_layer(self.h, i, _p(d)))
            out.append(tuple(int(v) for v in d))
        return out

    def weights(self, i: int):
        """-> weights [rows, K] ((ky, kx, cin) order along K), bias [rows]; bf16-representable float32"""
        _, rows, _, _, _, K = self.layers()[i]
        w = np.zeros((rows, K), np.float32); b = np.zeros(rows, np.float32)
        self._ck(self.L.mf_detector_get_weights(self.h, int(i), _p(w), _p(b)))
        return w, b

    def loadWeights(self, path: str):
        """mrcnn_class_*, mrcnn_bbox_fc and mrcnn_mask* of a safetensors weight file; all or nothing, complete on return (also between
        frames while the detector is attached to a context)"""
        self._ck(self.L.mf_detector_load_weights(self.h, os.fsencode(path)))
        return self

    def fcOutputs(self):
        """FC1 and FC2 outputs [1000, 1024] as float32 (bf16 values)"""
        a = np.zeros((self.ROIS, 1024), np.uint16); b = np.zeros((self.ROIS, 1024), np.uint16)
        self._ck(self.L.mf_detector_get_fc(self.h, _p(a), _p(b)))
        return _bf16_to_f32(a), _bf16_to_f32(b)

    def headOutputs(self):
        """fp32 (logits [1000, 81], deltas [1000, 81, 4])"""
        lg = np.zeros((self.ROIS, self.NUM_CLASSES), np.float32); dl = np.zeros((self.ROIS, self.NUM_CLASSES, 4), np.float32)
        self._ck(self.L.mf_detector_get_head_outputs(self.h, _p(lg), _p(dl)))
        return lg, dl

    def maskLayer(self, i: int) -> np.ndarray:
        """0 pooled [100, 14, 14, 256], 1..4 conv outputs [100, 14, 14, 256], 5 transposed conv [100, 14, 14, 2, 2, 256] (bf16 values as
        float32); 6 mask logits [100, 14, 14, 2, 2, 81] float32"""
        if i == 6:
            out = np.zeros((self.MAX_DETECTIONS, 14, 14, 2, 2, self.NUM_CLASSES), np.float32)
            self._ck(self.L.mf_detector_get_mask_layer(self.h, 6, _p(out)))
            return out
        raw = np.zeros((self.MAX_DETECTIONS, 14, 14, 2, 2, 256) if i == 5 else (self.MAX_DETECTIONS, 14, 14, 256), np.uint16)
        self._ck(self.L.mf_detector_get_mask_layer(self.h, int(i), _p(raw)))
        return _bf16_to_f32(raw)

    def detections(self):
        """-> (count, detections [100, 6] y1 x1 y2 x2 class score, zero rows past the count)"""
        d = np.zeros((self.MAX_DETECTIONS, 6), np.float32)
        n = self._ck(self.L.mf_detector_get_detections(self.h, _p(d)))
        return n, d

    def masks(self) -> np.ndarray:
        m = np.zeros((self.MAX_DETECTIONS, self.MASK, self.MASK), np.float32)
        self._ck(self.L.mf_detector_get_masks(self.h, _p(m)))
        return m

    def idImage(self):
        """-> (id_image H x W uint8, class ids, rois), the types of generate_id_image"""
        w, hh = C.c_int(0), C.c_int(0)
        self._ck(self.L.mf_detector_image_size(self.h, C.byref(w), C.byref(hh)))
        img = np.zeros((hh.value, w.value), np.uint8); ec = np.zeros(self.MAX_DETECTIONS, np.int32)
        er = np.zeros((self.MAX_DETECTIONS, 4), np.int32)
        n = self._ck(self.L.mf_detector_get_id_image(self.h, _p(img), _p(ec), _p(er)))
        return img, ec[:n].tolist(), er[:n].tolist()

    def execute(self, rgb: np.ndarray):
        """MaskRCNN.execute(): H x W x 3 uint8 RGB -> (id_image H x W uint8, class ids, rois), as generate_id_image returns them"""
        import torch
        a = np.ascontiguousarray(rgb, np.uint8)
        if a.ndim != 3 or a.shape[2] != 3:
            raise MFError("rgb must be HxWx3 uint8")
        H, W = a.shape[:2]
        rgba = torch.from_numpy(np.concatenate([a, np.full((H, W, 1), 255, np.uint8)], axis=2)).cuda()
        torch.cuda.current_stream().synchronize()          # the upload is complete before the detector's stream reads it
        self.detect(rgba.data_ptr(), W, H)
        out = self.idImage()                      # waits for the stream, so the upload outlives its use
        del rgba
        return out


def load_mask_rcnn(path: str, input_size: int = 1024, stream: int | None = None):
    """the reference's model.load_weights(COCO_MODEL_PATH, by_name=True): a Backbone, RegionProposals and Detector on `stream` with the
    weights of a safetensors file (scripts/convert_mrcnn_h5.py converts matterport's mask_rcnn_coco.h5) -> (backbone, rpn, detector).
    Close them in the reverse order."""
    made = []
    try:
        made.append(Backbone(input_size, stream=stream).loadWeights(path))
        made.append(RegionProposals(made[0]).loadWeights(path))
        made.append(Detector(made[1]).loadWeights(path))
    except BaseException:
        for h in reversed(made):
            h.close()
        raise
    return tuple(made)


def read_mrcnn_layer(path: str, layer: str):
    """one handle layer as the loaders fold it, on the host (no CUDA device): -> (weights [rows, K], bias [rows]), float32, zero padded.
    layer: a Keras conv layer name ("conv1", "res3a_branch2b", "fpn_p2", "mrcnn_mask_deconv", ...) or one of the stacked pairs
    "rpn_class_raw+rpn_bbox_pred", "mrcnn_class_logits+mrcnn_bbox_fc" (include/maskfusion_b200.h, mf_mrcnn_read_layer)"""
    L = load_library()
    dims = np.zeros(2, np.int32)
    if L.mf_mrcnn_read_layer(os.fsencode(path), layer.encode(), None, None, _p(dims)) != 0:
        raise _error()
    w = np.zeros((int(dims[0]), int(dims[1])), np.float32); b = np.zeros(int(dims[0]), np.float32)
    if L.mf_mrcnn_read_layer(os.fsencode(path), layer.encode(), _p(w), _p(b), _p(dims)) != 0:
        raise _error()
    return w, b
