"""Value types of the limap operator surface (host-side mirror of limap._limap._base).

Mirrors the pybind classes of src/limap/base/bindings.cc:132-284,433-524,688-1316 with the same names,
constructor overloads, fields and dict (pickle) layouts, so that loaders and runners written against
`limap.base` keep working: Line2d / Line3d (base/linebase.h:17-61), Camera / CameraPose / CameraImage /
CameraView (base/camera.h:33-112, base/camera_view.h), ImageCollection (base/image_collection.h),
LineTrack (base/linetrack.h:19-57), LineLinker{2d,3d}Config (base/line_linker.h). Only the two undistorted
pinhole models are legal on the triangulation / refinement path (base/camera_models.h:29-44), so COLMAP is
not needed. These are plain containers: the arithmetic of the hot path runs in the CUDA engine.
"""
import numpy as np

from .config import LINKER2D_DEFAULTS, LINKER3D_DEFAULTS

EPS = 1e-12  # util/types.h:34
MODEL_NAMES = {0: "SIMPLE_PINHOLE", 1: "PINHOLE"}
MODEL_IDS = {v: k for k, v in MODEL_NAMES.items()}


def _v(x, n):
    a = np.asarray(x, dtype=np.float64).reshape(-1)
    if a.size != n:
        raise ValueError(f"expected {n} values, got {a.size}")
    return a.copy()


def _normalized(v):
    n2 = float(np.dot(v, v))
    return v / np.sqrt(n2) if n2 > 0 else v  # Eigen normalized()


class Line2d:
    """base/linebase.h:17-37"""

    def __init__(self, *args, score=-1.0):
        if len(args) == 0:
            self.start, self.end = np.zeros(2), np.zeros(2)
        elif len(args) == 1:
            seg = np.asarray(args[0], dtype=np.float64)
            if seg.shape != (2, 2):
                raise RuntimeError("THROW_CHECK_EQ(seg.rows(), 2) / (seg.cols(), 2)")
            self.start, self.end = seg[0].copy(), seg[1].copy()
        else:
            self.start, self.end = _v(args[0], 2), _v(args[1], 2)
            if len(args) > 2:
                score = args[2]
        self.score = float(score)

    def length(self):
        return float(np.linalg.norm(self.start - self.end))

    def midpoint(self):
        return 0.5 * (self.start + self.end)

    def direction(self):
        return _normalized(self.end - self.start)

    def perp_direction(self):
        d = self.direction()
        return np.array([d[1], -d[0]])

    def coords(self):
        return _normalized(np.cross(np.append(self.start, 1.0), np.append(self.end, 1.0)))

    def point_projection(self, p):
        p = _v(p, 2)
        proj = float(np.dot(p - self.start, self.direction()))
        if proj < 0:
            return self.start.copy()
        if proj > self.length():
            return self.end.copy()
        return self.start + proj * self.direction()

    def point_distance(self, p):
        return float(np.linalg.norm(_v(p, 2) - self.point_projection(p)))

    def as_array(self):
        return np.stack([self.start, self.end])

    def __repr__(self):
        return f"Line2d({self.start.tolist()}, {self.end.tolist()})"


class Line3d:
    """base/linebase.h:39-61"""

    def __init__(self, *args, score=-1.0, depth_start=-1.0, depth_end=-1.0, uncertainty=-1.0):
        if len(args) == 0:
            self.start, self.end = np.zeros(3), np.zeros(3)
        elif len(args) == 1:
            seg = np.asarray(args[0], dtype=np.float64)
            if seg.shape != (2, 3):
                raise RuntimeError("THROW_CHECK_EQ(seg.rows(), 2) / (seg.cols(), 3)")
            self.start, self.end = seg[0].copy(), seg[1].copy()
        else:
            self.start, self.end = _v(args[0], 3), _v(args[1], 3)
            rest = list(args[2:])
            if rest:
                score = rest.pop(0)
            if rest:
                depth_start = rest.pop(0)
            if rest:
                depth_end = rest.pop(0)
            if rest:
                uncertainty = rest.pop(0)
        self.score = float(score)
        self.uncertainty = float(uncertainty)
        self.depths = np.array([float(depth_start), float(depth_end)])

    def set_uncertainty(self, val):
        self.uncertainty = float(val)

    def length(self):
        return float(np.linalg.norm(self.start - self.end))

    def midpoint(self):
        return 0.5 * (self.start + self.end)

    def direction(self):
        return _normalized(self.end - self.start)

    def as_array(self):
        return np.stack([self.start, self.end])

    def projection(self, view):
        return Line2d(view.projection(self.start), view.projection(self.end))

    def sensitivity(self, view):  # base/linebase.cc:100-107
        l2 = self.projection(view)
        d3 = view.ray_direction(l2.midpoint())
        c = abs(float(np.dot(self.direction(), d3)))
        return 90.0 - np.degrees(np.arccos(c))

    def computeUncertainty(self, view, var2d=5.0):  # base/linebase.cc:109-116
        d = 0.5 * (view.pose.projdepth(self.start) + view.pose.projdepth(self.end))
        return view.cam.uncertainty(d, var2d)

    def __repr__(self):
        return f"Line3d({self.start.tolist()}, {self.end.tolist()})"


class LineList(list):
    """list[Line2d] that remembers the (N, 4) array it came from, so that Init() can hand the segments to
    the engine without walking 1e5 Python objects."""
    array = None


def _GetLine2dVectorFromArray(segs2d):  # base/linebase.cc:130-139
    a = np.asarray(segs2d, dtype=np.float64)
    if a.ndim != 2 or (a.shape[0] != 0 and a.shape[1] < 4):
        raise RuntimeError("THROW_CHECK_GE(segs2d.cols(), 4)")
    out = LineList(Line2d(r[0:2], r[2:4]) for r in a)
    out.array = np.ascontiguousarray(a[:, :4]) if len(a) else np.zeros((0, 4))
    return out


def _GetLine3dVectorFromArray(segs3d):
    return [Line3d(np.asarray(s)) for s in segs3d]


def get_all_lines_2d(all_2d_segs):  # base/functions.py:4-24
    return {img_id: _GetLine2dVectorFromArray(segs) for img_id, segs in all_2d_segs.items()}


def get_all_lines_3d(all_3d_segs):  # base/functions.py:27-47
    return {img_id: _GetLine3dVectorFromArray(s) for img_id, s in all_3d_segs.items()}


def get_invert_idmap_from_linetracks(all_lines_2d, linetracks):  # base/functions.py:50-72
    m = {img_id: [-1] * len(lines) for img_id, lines in all_lines_2d.items()}
    for track_id, track in enumerate(linetracks):
        for img_id, line_id in zip(track.image_id_list, track.line_id_list):
            m[img_id][line_id] = track_id
    return m


def _quat_to_R(q):  # base/pose.cc:12-29 (Eigen toRotationMatrix of the normalised quaternion)
    q = np.asarray(q, dtype=np.float64)
    n = np.linalg.norm(q)
    q = np.array([1.0, q[1], q[2], q[3]]) if n == 0 else q / n
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _R_to_quat(R):  # Eigen Quaterniond(Matrix3d)
    from .synth import _rot_to_quat
    return _rot_to_quat(np.asarray(R, dtype=np.float64))


class Camera:
    """base/camera.h:33-87 for the two undistorted pinhole models."""

    def __init__(self, *args, cam_id=-1, hw=(-1, -1)):
        self.model_id, self.params, self.cam_id = 1, [], int(cam_id)
        self.height, self.width = int(hw[0]), int(hw[1])
        self.initialized = []
        if len(args) == 0:
            return
        if len(args) == 1 and isinstance(args[0], dict):
            d = args[0]
            self.model_id = int(d["model_id"])
            self.params = [float(x) for x in d["params"]]
            self.cam_id = int(d["cam_id"])
            self.height, self.width = int(d["height"]), int(d["width"])
            self.initialized = list(d.get("initialized", [True] * len(self.params)))
            self._check()
            return
        if len(args) == 1 and isinstance(args[0], Camera):
            o = args[0]
            self.model_id, self.params, self.cam_id = o.model_id, list(o.params), o.cam_id
            self.height, self.width, self.initialized = o.height, o.width, list(o.initialized)
            return
        a = list(args)
        first = a.pop(0)
        if isinstance(first, str):
            if first not in MODEL_IDS:
                raise RuntimeError("Camera model does not exist")  # only undistorted models on this path
            self.model_id = MODEL_IDS[first]
        elif np.isscalar(first):
            self.model_id = int(first)
        else:  # Camera(K, cam_id, hw): PINHOLE from a calibration matrix
            self.model_id = 1
            a.insert(0, first)
        if a and not np.isscalar(a[0]):
            p = np.asarray(a.pop(0), dtype=np.float64)
            if p.shape == (3, 3):
                K = p
                self.params = ([K[0, 0], K[0, 2], K[1, 2]] if self.model_id == 0
                               else [K[0, 0], K[1, 1], K[0, 2], K[1, 2]])
            else:
                self.params = [float(x) for x in p.reshape(-1)]
        if a:
            self.cam_id = int(a.pop(0))
        if a:
            hw = a.pop(0)
            self.height, self.width = int(hw[0]), int(hw[1])
        self.initialized = [True] * len(self.params)
        self._check()

    def _check(self):
        if self.model_id not in MODEL_NAMES:
            raise RuntimeError("Error! Limap optimization does not support non-pinhole models.")
        if self.params and len(self.params) != (3 if self.model_id == 0 else 4):
            raise RuntimeError("THROW_CHECK(VerifyParams())")

    def model_name(self):
        return MODEL_NAMES[self.model_id]

    def resize(self, width, height):  # colmap Camera::Rescale(width, height) (base/camera.h:69-71)
        sx, sy = width / float(self.width), height / float(self.height)
        self.width, self.height = int(width), int(height)
        p = self.params
        if self.model_id == 0:
            self.params = [p[0] * (sx + sy) / 2.0, p[1] * sx, p[2] * sy]
        else:
            self.params = [p[0] * sx, p[1] * sy, p[2] * sx, p[3] * sy]

    def set_max_image_dim(self, val):  # base/camera.cc:216-226
        if val <= 0:
            raise RuntimeError("THROW_CHECK_GT(val, 0)")
        ratio = float(val) / float(max(self.height, self.width))
        if ratio < 1.0:
            # C round(): halves away from zero (Python's round() goes to the even neighbour)
            self.resize(int(np.floor(ratio * self.width + 0.5)), int(np.floor(ratio * self.height + 0.5)))

    def kvec(self):  # base/camera_models.h:29-44 ParamsToKvec
        p = self.params
        return np.array([p[0], p[0], p[1], p[2]] if self.model_id == 0 else [p[0], p[1], p[2], p[3]])

    def K(self):
        fx, fy, cx, cy = self.kvec()
        return np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1.0]])

    def K_inv(self):
        return np.linalg.inv(self.K())

    def h(self):
        return self.height

    def w(self):
        return self.width

    def IsUndistorted(self):
        return True

    def uncertainty(self, depth, var2d=5.0):  # base/camera.cc:228-242
        f = self.params[0] if self.model_id == 0 else 0.5 * (self.params[0] + self.params[1])
        return var2d * depth / f

    def as_dict(self):  # base/camera.cc:266-274
        return {"model_id": self.model_id, "params": list(self.params), "cam_id": self.cam_id,
                "height": self.height, "width": self.width, "initialized": list(self.initialized)}


class CameraPose:
    """base/camera.h:89-112"""

    def __init__(self, *args, initialized=None):
        self.qvec, self.tvec, self.initialized = np.array([1.0, 0, 0, 0]), np.zeros(3), False
        if len(args) == 1 and isinstance(args[0], dict):
            d = args[0]
            self.qvec = _normalized(_v(d["qvec"], 4))
            self.tvec = _v(d["tvec"], 3)
            self.initialized = bool(d.get("initialized", True))
        elif len(args) == 1 and isinstance(args[0], CameraPose):
            self.qvec, self.tvec, self.initialized = args[0].qvec.copy(), args[0].tvec.copy(), args[0].initialized
        elif len(args) >= 2:
            a0 = np.asarray(args[0], dtype=np.float64)
            self.qvec = _R_to_quat(a0) if a0.shape == (3, 3) else _normalized(_v(a0, 4))
            self.tvec = _v(args[1], 3)
            self.initialized = bool(args[2]) if len(args) > 2 else True
        elif len(args) == 1:
            self.initialized = bool(args[0])
        if initialized is not None:
            self.initialized = bool(initialized)

    def R(self):
        return _quat_to_R(self.qvec)

    def T(self):
        return self.tvec

    def center(self):
        return -self.R().T @ self.tvec

    def projdepth(self, p3d):
        return float((self.R() @ _v(p3d, 3) + self.tvec)[2])

    def SetInitFlag(self, flag):
        self.initialized = bool(flag)

    def as_dict(self):
        return {"qvec": self.qvec.copy(), "tvec": self.tvec.copy(), "initialized": self.initialized}


class CameraImage:
    """base/camera_view.h CameraImage(cam_id | camera, pose, image_name)"""

    def __init__(self, *args):
        if len(args) == 1 and isinstance(args[0], dict):
            d = args[0]
            self.cam_id, self.pose, self._name = int(d["cam_id"]), CameraPose(d["pose"]), d.get("image_name", "none")
            return
        cam = args[0]
        self.cam_id = cam.cam_id if isinstance(cam, Camera) else int(cam)
        self.pose = args[1] if len(args) > 1 and isinstance(args[1], CameraPose) else CameraPose()
        self._name = args[-1] if isinstance(args[-1], str) else "none"

    def image_name(self):
        return self._name

    def SetImageName(self, name):
        self._name = name

    def as_dict(self):
        return {"cam_id": self.cam_id, "pose": self.pose.as_dict(), "image_name": self._name}


class CameraView:
    """base/camera_view.h:44-88, base/camera_view.cc:53-82"""

    def __init__(self, *args):
        if len(args) == 1 and isinstance(args[0], dict):
            d = args[0]
            self.cam, self.pose, self._name = Camera(d["camera"]), CameraPose(d["pose"]), d.get("image_name", "none")
            return
        self.cam = args[0]
        self.pose = args[1] if len(args) > 1 and isinstance(args[1], CameraPose) else CameraPose()
        self._name = args[-1] if isinstance(args[-1], str) else "none"

    def image_name(self):
        return self._name

    def K(self):
        return self.cam.K()

    def K_inv(self):
        return self.cam.K_inv()

    def R(self):
        return self.pose.R()

    def T(self):
        return self.pose.T()

    def h(self):
        return self.cam.h()

    def w(self):
        return self.cam.w()

    def matrix(self):
        return self.K() @ np.concatenate([self.R(), self.T()[:, None]], axis=1)

    def projection(self, p3d):
        ph = self.K() @ (self.R() @ _v(p3d, 3) + self.T())
        return ph[:2] / (ph[2] + EPS)

    def ray_direction(self, p2d):
        p = _v(p2d, 2)
        return _normalized((self.R().T @ self.K_inv()) @ np.array([p[0], p[1], 1.0]))

    def get_direction_from_vp(self, vp):
        return _normalized((self.R().T @ self.K_inv()) @ _v(vp, 3))

    def as_dict(self):
        return {"camera": self.cam.as_dict(), "pose": self.pose.as_dict(), "image_name": self._name}


class ImageCollection:
    """base/image_collection.h: cameras {cam_id: Camera} + images {img_id: CameraImage}."""

    def __init__(self, *args):
        self.cameras, self.images = {}, {}
        if len(args) == 1 and isinstance(args[0], dict):  # as_dict layout (image_collection.cc:158-171)
            d = args[0]
            self.cameras = {int(k): Camera(v) for k, v in d["cameras"].items()}
            self.images = {int(k): CameraImage(v) for k, v in d["images"].items()}
        elif len(args) == 1 and isinstance(args[0], ImageCollection):
            self.cameras = {k: Camera(v) for k, v in args[0].cameras.items()}
            self.images = {k: CameraImage(v.as_dict()) for k, v in args[0].images.items()}
        elif len(args) == 1:  # list[CameraView]
            for i, view in enumerate(args[0]):
                cam = Camera(view.cam)
                cam.cam_id = i
                self.cameras[i] = cam
                self.images[i] = CameraImage(i, view.pose, view.image_name())
        elif len(args) == 2:
            cams, imgs = args
            self.cameras = dict(cams) if isinstance(cams, dict) else {c.cam_id: c for c in cams}
            self.images = dict(imgs) if isinstance(imgs, dict) else {i: im for i, im in enumerate(imgs)}

    def NumCameras(self):
        return len(self.cameras)

    def NumImages(self):
        return len(self.images)

    def get_cam_ids(self):
        return sorted(self.cameras)

    def get_img_ids(self):
        return sorted(self.images)

    def get_cameras(self):
        return [self.cameras[k] for k in self.get_cam_ids()]

    def get_images(self):
        return [self.images[k] for k in self.get_img_ids()]

    def exist_cam(self, cam_id):
        return cam_id in self.cameras

    def exist_image(self, img_id):
        return img_id in self.images

    def cam(self, cam_id):
        return self.cameras[cam_id]

    def camimage(self, img_id):
        return self.images[img_id]

    def campose(self, img_id):
        return self.images[img_id].pose

    def camview(self, img_id):
        im = self.images[img_id]
        return CameraView(self.cameras[im.cam_id], im.pose, im.image_name())

    def image_name(self, img_id):
        return self.images[img_id].image_name()

    def get_camviews(self):
        return [self.camview(i) for i in self.get_img_ids()]

    def get_map_camviews(self):
        return {i: self.camview(i) for i in self.get_img_ids()}

    def get_locations(self):
        return [self.campose(i).center() for i in self.get_img_ids()]

    def IsUndistorted(self):
        return all(c.IsUndistorted() for c in self.cameras.values())

    def set_max_image_dim(self, val):  # base/image_collection.cc: every camera
        for c in self.cameras.values():
            c.set_max_image_dim(val)

    def get_image_name_dict(self):
        return {i: self.images[i].image_name() for i in self.get_img_ids()}

    def update_neighbors(self, neighbors):  # base/image_collection.cc:322-342
        if len(neighbors) == self.NumImages():
            return neighbors
        out = {}
        for i in self.get_img_ids():
            if i not in neighbors:
                raise RuntimeError("Error! The image id is not found in the input neighbors.")
            out[i] = [j for j in neighbors[i] if self.exist_image(j)]
        return out

    def as_dict(self):
        return {"cameras": {k: v.as_dict() for k, v in self.cameras.items()},
                "images": {k: v.as_dict() for k, v in self.images.items()}}

    def arrays(self):
        """(img_ids, model_ids, kvec[V,4], qvec[V,4], tvec[V,3]) in ascending image id order."""
        ids = self.get_img_ids()
        V = len(ids)
        model, kvec, qvec, tvec = np.zeros(V, np.int32), np.zeros((V, 4)), np.zeros((V, 4)), np.zeros((V, 3))
        for v, i in enumerate(ids):
            im = self.images[i]
            cam = self.cameras[im.cam_id]
            model[v], kvec[v], qvec[v], tvec[v] = cam.model_id, cam.kvec(), im.pose.qvec, im.pose.tvec
        return np.asarray(ids, np.int32), model, kvec, qvec, tvec


class LineTrack:
    """base/linetrack.h:19-57"""

    def __init__(self, *args):
        self.line = Line3d()
        self.image_id_list, self.line_id_list, self.line2d_list = [], [], []
        self.node_id_list, self.line3d_list, self.score_list = [], [], []
        self.active = True
        if len(args) == 1 and isinstance(args[0], LineTrack):
            o = args[0]
            self.line = Line3d(o.line.start, o.line.end, o.line.score, o.line.depths[0], o.line.depths[1],
                               o.line.uncertainty)
            self.image_id_list, self.line_id_list = list(o.image_id_list), list(o.line_id_list)
            self.line2d_list, self.node_id_list = list(o.line2d_list), list(o.node_id_list)
            self.line3d_list, self.score_list, self.active = list(o.line3d_list), list(o.score_list), o.active
        elif len(args) == 1 and isinstance(args[0], dict):
            d = args[0]
            self.line = Line3d(np.asarray(d["line"])) if not isinstance(d["line"], Line3d) else d["line"]
            self.image_id_list, self.line_id_list = list(d["image_id_list"]), list(d["line_id_list"])
            self.line2d_list = [x if isinstance(x, Line2d) else Line2d(np.asarray(x)) for x in d["line2d_list"]]
            self.node_id_list = list(d.get("node_id_list", []))
            self.line3d_list = [x if isinstance(x, Line3d) else Line3d(np.asarray(x))
                                for x in d.get("line3d_list", [])]
            self.score_list = list(d.get("score_list", []))
        elif len(args) == 4:
            self.line, self.image_id_list, self.line_id_list, self.line2d_list = (
                args[0], list(args[1]), list(args[2]), list(args[3]))

    def count_lines(self):
        return len(self.line2d_list)

    def GetSortedImageIds(self):
        return sorted(set(self.image_id_list))

    def count_images(self):
        return len(set(self.image_id_list))

    def GetIdMap(self):
        m = {}
        for k, i in enumerate(self.image_id_list):
            m.setdefault(i, []).append(k)
        return m

    def GetIndexMapforSorted(self):
        return {i: k for k, i in enumerate(self.GetSortedImageIds())}

    def GetIndexesforSorted(self):
        m = self.GetIndexMapforSorted()
        return [m[i] for i in self.image_id_list]

    def HasImage(self, image_id):
        return image_id in self.image_id_list

    def Resize(self, n_lines):  # base/linetrack.cc Resize
        self.image_id_list, self.line_id_list = [0] * n_lines, [0] * n_lines
        self.line2d_list = [Line2d() for _ in range(n_lines)]
        self.node_id_list, self.score_list = [0] * n_lines, [0.0] * n_lines
        self.line3d_list = [Line3d() for _ in range(n_lines)]

    def Write(self, filename):
        """base/linetrack.cc:133-213 (std::fixed, setprecision(10); NaN endpoints are written as 0)."""
        ff = lambda v: f"{float(v):.10f}"
        n_lines = self.count_lines()
        with open(filename, "w") as f:
            row = ""
            for v in list(self.line.start) + list(self.line.end):
                row += (ff(0.0) if np.isnan(v) else ff(v)) + " "
            f.write(row + "\n")
            f.write(f"{n_lines} {self.count_images()}\n")
            f.write("image_id_list " + "".join(f"{int(i)} " for i in self.image_id_list) + "\n")
            f.write("line_id_list " + "".join(f"{int(i)} " for i in self.line_id_list) + "\n")
            f.write("line2d_list\n")
            for l in self.line2d_list:
                f.write(f"{ff(l.start[0])} {ff(l.start[1])} {ff(l.end[0])} {ff(l.end[1])} \n")
            if self.node_id_list:
                f.write("node_id_list " + "".join(f"{int(i)} " for i in self.node_id_list) + "\n")
            if self.score_list:
                f.write("score_list " + "".join(f"{ff(x)} " for x in self.score_list) + "\n")
            if self.line3d_list:
                f.write("line3d_list\n")
                for l in self.line3d_list:
                    f.write("".join(f"{ff(v)} " for v in list(l.start) + list(l.end)) + "\n")
            f.write("END\n")

    def Read(self, filename):
        """base/linetrack.cc:215-270 (token stream like operator>>)."""
        with open(filename) as f:
            tok = f.read().split()
        p = 0

        def take(n, conv):
            nonlocal p
            out = [conv(x) for x in tok[p:p + n]]
            p += n
            return out

        v = take(6, float)
        self.line = Line3d(np.array(v[:3]), np.array(v[3:]))
        n_lines, _ = take(2, int)
        self.Resize(n_lines)
        if take(1, str) != ["image_id_list"]:
            raise RuntimeError("THROW_CHECK_EQ(str, \"image_id_list\")")
        self.image_id_list = take(n_lines, int)
        if take(1, str) != ["line_id_list"]:
            raise RuntimeError("THROW_CHECK_EQ(str, \"line_id_list\")")
        self.line_id_list = take(n_lines, int)
        if take(1, str) != ["line2d_list"]:  # files of the previous version stop here
            return
        for i in range(n_lines):
            a = take(4, float)
            self.line2d_list[i] = Line2d(np.array(a[:2]), np.array(a[2:]))
        s = take(1, str)
        if s == ["END"] or not s:
            return
        if s != ["node_id_list"]:
            raise RuntimeError("THROW_CHECK_EQ(str, \"node_id_list\")")
        self.node_id_list = take(n_lines, int)
        if take(1, str) != ["score_list"]:
            raise RuntimeError("THROW_CHECK_EQ(str, \"score_list\")")
        self.score_list = take(n_lines, float)
        if take(1, str) != ["line3d_list"]:
            raise RuntimeError("THROW_CHECK_EQ(str, \"line3d_list\")")
        for i in range(n_lines):
            a = take(6, float)
            self.line3d_list[i] = Line3d(np.array(a[:3]), np.array(a[3:]))

    def as_dict(self):
        return {"line": self.line.as_array(), "image_id_list": list(self.image_id_list),
                "line_id_list": list(self.line_id_list), "line2d_list": [l.as_array() for l in self.line2d_list],
                "node_id_list": list(self.node_id_list), "line3d_list": [l.as_array() for l in self.line3d_list],
                "score_list": list(self.score_list)}


class PatchNode:
    """base/graph.h:37-46 (read-only view of one node of a Graph)."""

    def __init__(self, image_idx, line_idx, node_idx):
        self.image_idx, self.line_idx, self.node_idx = int(image_idx), int(line_idx), int(node_idx)


class Edge:
    """base/graph.h:25-35 (read-only view of one undirected edge of a Graph)."""

    def __init__(self, node_idx1, node_idx2, sim, edge_idx):
        self.node_idx1, self.node_idx2, self.sim, self.edge_idx = int(node_idx1), int(node_idx2), float(sim), int(edge_idx)

    @property
    def similarity(self):
        return self.sim


class Graph:
    """base/graph.h:48-67 as base/bindings.cc:58-68 exposes it, read-only and backed by arrays: node i is
    (image_idx[i], line_idx[i]); edge e is (node1[e], node2[e], sim[e]) in insertion order. Node and edge objects are
    built on access."""

    def __init__(self, image_idx=(), line_idx=(), node1=(), node2=(), sim=()):
        self.image_idx = np.asarray(image_idx, np.int64)
        self.line_idx = np.asarray(line_idx, np.int64)
        self.node1 = np.asarray(node1, np.int64)
        self.node2 = np.asarray(node2, np.int64)
        self.sim = np.asarray(sim, np.float64)

    @property
    def nodes(self):
        return [PatchNode(i, l, k) for k, (i, l) in enumerate(zip(self.image_idx.tolist(), self.line_idx.tolist()))]

    @property
    def undirected_edges(self):
        return [Edge(a, b, w, e) for e, (a, b, w) in enumerate(zip(self.node1.tolist(), self.node2.tolist(),
                                                                  self.sim.tolist()))]

    @property
    def node_map(self):
        return {(i, l): k for k, (i, l) in enumerate(zip(self.image_idx.tolist(), self.line_idx.tolist()))}

    def get_node_id(self, image_idx, line_idx):  # graph.cc:72-78: size_t(-1) when absent
        return self.node_map.get((int(image_idx), int(line_idx)), 2 ** 64 - 1)

    def _endpoints(self):
        # AddEdge appends the edge to out_edges and in_edges of both ends (graph.cc:18-21, :80-86)
        ends = np.empty(2 * len(self.node1), np.int64)
        ends[0::2], ends[1::2] = self.node1, self.node2
        return ends

    @property
    def input_degrees(self):
        return np.bincount(self._endpoints(), minlength=len(self.image_idx)).tolist()

    @property
    def output_degrees(self):
        return self.input_degrees

    @property
    def scores(self):  # graph.cc:45-55: sum of the out-edge similarities, added in insertion order
        s = np.zeros(len(self.image_idx))
        np.add.at(s, self._endpoints(), np.repeat(self.sim, 2))
        return [(float(x), k) for k, x in enumerate(s.tolist())]


class _LinkerConfig:
    _defaults = {}

    def __init__(self, d=None):
        for k, v in self._defaults.items():
            setattr(self, k, v)
        for k, v in (d or {}).items():
            if k in self._defaults:
                setattr(self, k, v)

    def as_dict(self):
        return {k: getattr(self, k) for k in self._defaults}


class LineLinker2dConfig(_LinkerConfig):
    _defaults = {k: v for k, v in LINKER2D_DEFAULTS.items() if k != "th_scaleinv" and k != "use_scaleinv"}


class LineLinker3dConfig(_LinkerConfig):
    _defaults = dict(LINKER3D_DEFAULTS)

    def set_to_shared_parent_scoring(self):
        self.use_angle, self.use_overlap, self.use_perp, self.use_innerseg, self.use_scaleinv = True, False, False, False, True

    def set_to_spatial_merging(self):
        self.use_angle, self.use_overlap, self.use_perp, self.use_innerseg, self.use_scaleinv = True, True, False, True, False


class LineLinker2d:
    def __init__(self, cfg=None):
        self.config = cfg if isinstance(cfg, LineLinker2dConfig) else LineLinker2dConfig(cfg)


class LineLinker3d:
    def __init__(self, cfg=None):
        self.config = cfg if isinstance(cfg, LineLinker3dConfig) else LineLinker3dConfig(cfg)


class LineLinker:
    def __init__(self, cfg2d=None, cfg3d=None):
        self.linker_2d, self.linker_3d = LineLinker2d(cfg2d), LineLinker3d(cfg3d)

    def GetLinker2d(self):
        return self.linker_2d

    def GetLinker3d(self):
        return self.linker_3d
