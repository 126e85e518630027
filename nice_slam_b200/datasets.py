"""Dataset readers (src/utils/datasets.py) with frame preparation on the GPU.

The file lists and poses restate the reference's for 'replica', 'scannet', 'azure' and 'tumrgbd'.  Frames are decoded on the host with
cv2.imread, the reference's decoder, so the bytes are the same: colour BGR u8, depth u16 (IMREAD_UNCHANGED).  A background thread
decodes up to `prefetch` frames ahead into pinned staging buffers; the raw bytes go to the device on a side stream, and an event orders
the upload before nsb_frame_prepare, which computes the reference's undistort / colour conversion / resize / crop chain
(include/nice_slam_b200.h, "frame preparation").  Items are (idx, colour f64 [H,W,3], depth f32 [H,W], c2w f32 [4,4]) with colour and
depth on the device, which FusedSLAM.run takes as they are.

Deviation: the reference scales a pose's translation by `scale` inside __getitem__, on the stored pose, so a frame read twice is scaled
twice when scale != 1; here the poses are scaled once, when they are loaded.  (Every shipped config has scale 1.)"""
import glob
import os
import queue
import threading

import cv2
import numpy as np
import torch

from . import _lib
from .cull import load_poses


def _flip(c2w):
    c2w[:3, 1] *= -1
    c2w[:3, 2] *= -1
    return c2w


def replica_files(folder):
    color = sorted(glob.glob(f"{folder}/results/frame*.jpg"))
    depth = sorted(glob.glob(f"{folder}/results/depth*.png"))
    poses = [torch.from_numpy(p).float() for p in load_poses(f"{folder}/traj.txt")[:len(color)]]
    return color, depth, poses


def scannet_files(folder):
    folder = os.path.join(folder, "frames")
    stem = lambda x: int(os.path.basename(x)[:-4])      # noqa: E731
    color = sorted(glob.glob(os.path.join(folder, "color", "*.jpg")), key=stem)
    depth = sorted(glob.glob(os.path.join(folder, "depth", "*.png")), key=stem)
    poses = []
    for path in sorted(glob.glob(os.path.join(folder, "pose", "*.txt")), key=stem):
        with open(path, "r") as f:
            rows = [list(map(float, line.split(" "))) for line in f.readlines()]
        poses.append(torch.from_numpy(_flip(np.array(rows).reshape(4, 4))).float())
    return color, depth, poses


def azure_files(folder):
    color = sorted(glob.glob(os.path.join(folder, "color", "*.jpg")))
    depth = sorted(glob.glob(os.path.join(folder, "depth", "*.png")))
    path = os.path.join(folder, "scene", "trajectory.log")
    poses = []
    if os.path.exists(path):
        with open(path) as f:
            content = f.readlines()
        for i in range(0, len(content), 5):
            c2w = np.array(list(map(float, ("".join(content[i + 1:i + 5])).strip().split()))).reshape((4, 4))
            poses.append(torch.from_numpy(_flip(c2w)).float())
    else:
        poses = [torch.from_numpy(np.eye(4)).float() for _ in color]
    return color, depth, poses


def _parse_list(path, skiprows=0):
    return np.loadtxt(path, delimiter=" ", dtype=str, skiprows=skiprows)


def tum_associate(tstamp_image, tstamp_depth, tstamp_pose, max_dt=0.08):
    """TUM_RGBD.associate_frames: (image, depth, pose) index triples whose depth and pose stamps lie within max_dt of the image's."""
    out = []
    for i, t in enumerate(tstamp_image):
        j = np.argmin(np.abs(tstamp_depth - t))
        k = np.argmin(np.abs(tstamp_pose - t))
        if (np.abs(tstamp_depth[j] - t) < max_dt) and (np.abs(tstamp_pose[k] - t) < max_dt):
            out.append((i, j, k))
    return out


def _pose_from_quaternion(pvec):
    from scipy.spatial.transform import Rotation
    pose = np.eye(4)
    pose[:3, :3] = Rotation.from_quat(pvec[3:]).as_matrix()
    pose[:3, 3] = pvec[:3]
    return pose


def tum_files(folder, frame_rate=32):
    """TUM_RGBD.loadtum: associations, subsampled to frame_rate, poses relative to the first."""
    pose_list = os.path.join(folder, "groundtruth.txt")
    if not os.path.isfile(pose_list):
        pose_list = os.path.join(folder, "pose.txt")
    image_data = _parse_list(os.path.join(folder, "rgb.txt"))
    depth_data = _parse_list(os.path.join(folder, "depth.txt"))
    pose_data = _parse_list(pose_list, skiprows=1)
    pose_vecs = pose_data[:, 1:].astype(np.float64)
    tstamp_image = image_data[:, 0].astype(np.float64)
    assoc = tum_associate(tstamp_image, depth_data[:, 0].astype(np.float64), pose_data[:, 0].astype(np.float64))
    keep = [0]
    for i in range(1, len(assoc)):
        if tstamp_image[assoc[i][0]] - tstamp_image[assoc[keep[-1]][0]] > 1.0 / frame_rate:
            keep.append(i)
    color, depth, poses, inv_pose = [], [], [], None
    for ix in keep:
        i, j, k = assoc[ix]
        color.append(os.path.join(folder, image_data[i, 1]))
        depth.append(os.path.join(folder, depth_data[j, 1]))
        c2w = _pose_from_quaternion(pose_vecs[k])
        if inv_pose is None:
            inv_pose = np.linalg.inv(c2w)
            c2w = np.eye(4)
        else:
            c2w = inv_pose @ c2w
        poses.append(torch.from_numpy(_flip(c2w)).float())
    return color, depth, poses


FILES = {"replica": replica_files, "scannet": scannet_files, "azure": azure_files, "tumrgbd": tum_files}


def frame_params(cfg, color_shape, depth_shape):
    """nsb_frame_params of cfg['cam'] for raw images of these [H, W]."""
    cam = cfg["cam"]
    p = _lib.FrameParams()
    p.color_h, p.color_w = int(color_shape[0]), int(color_shape[1])
    p.depth_h, p.depth_w = int(depth_shape[0]), int(depth_shape[1])
    p.fx, p.fy, p.cx, p.cy = (float(cam[k]) for k in ("fx", "fy", "cx", "cy"))
    dist = cam.get("distortion")
    p.undistort = int(dist is not None)
    if dist is not None:
        if len(dist) != 5:
            raise RuntimeError("cam.distortion: expected k1 k2 p1 p2 k3, got %d coefficients" % len(dist))
        for n, v in enumerate(dist):
            p.dist[n] = float(v)
    p.png_depth_scale, p.scale = float(cam["png_depth_scale"]), float(cfg["scale"])
    crop = cam.get("crop_size")
    p.crop_h, p.crop_w = (int(crop[0]), int(crop[1])) if crop is not None else (0, 0)
    p.crop_edge = int(cam["crop_edge"])
    return p


def prepare_frame(params, color_raw, depth_raw, stream=None):
    """nsb_frame_prepare on device tensors color_raw u8 [h,w,3] (BGR) and depth_raw int16-stored u16 [h,w] -> (colour f64, depth f32)."""
    L = _lib.lib()
    H, W = _lib.C.c_int(0), _lib.C.c_int(0)
    L.nsb_frame_output_size(_lib.C.byref(params), _lib.C.byref(H), _lib.C.byref(W))
    dev = color_raw.device
    color = torch.empty(H.value, W.value, 3, dtype=torch.float64, device=dev)
    depth = torch.empty(H.value, W.value, dtype=torch.float32, device=dev)
    nws = L.nsb_frame_workspace(_lib.C.byref(params))
    ws = torch.empty(max(nws, 1), dtype=torch.uint8, device=dev)
    s = stream if stream is not None else torch.cuda.current_stream(dev)
    _lib.check(L.nsb_frame_prepare(_lib.C.byref(params), color_raw.data_ptr(), depth_raw.data_ptr(), ws.data_ptr(), nws,
                                   color.data_ptr(), depth.data_ptr(), _lib.C.c_void_p(s.cuda_stream)), "nsb_frame_prepare")
    return color, depth


def decode(color_path, depth_path):
    """cv2.imread of one frame: (BGR u8 [h,w,3], depth u16 [h,w])."""
    color = cv2.imread(color_path)
    depth = cv2.imread(depth_path, cv2.IMREAD_UNCHANGED)
    if color is None or depth is None:
        raise RuntimeError("cannot read frame %s / %s" % (color_path, depth_path))
    if depth.dtype != np.uint16 or depth.ndim != 2:
        raise RuntimeError("%s: expected a single-channel 16-bit PNG, got %s %s" % (depth_path, depth.dtype, depth.shape))
    return color, depth


class FrameReader:
    """The frames of cfg['dataset'] under input_folder (default cfg['data']['input_folder']), prepared on `device`.  Iterating starts a
    decoder thread that stays `prefetch` frames ahead (0: decode in the caller's thread); the thread is joined when the iteration ends,
    raises or is abandoned.  len() and [idx] work as for the reference's dataset."""

    def __init__(self, cfg, input_folder=None, device="cuda:0", prefetch=2):
        name = cfg["dataset"]
        if name == "cofusion":
            raise RuntimeError("dataset 'cofusion' is not supported: its depth is OpenEXR, and no EXR reader is available")
        if name not in FILES:
            raise RuntimeError("unknown dataset %r (supported: %s)" % (name, ", ".join(sorted(FILES))))
        self.cfg, self.name, self.device, self.prefetch = cfg, name, torch.device(device), int(prefetch)
        self.input_folder = input_folder if input_folder is not None else cfg["data"]["input_folder"]
        self.color_paths, self.depth_paths, poses = FILES[name](self.input_folder)
        self.n_img = len(self.color_paths)
        if len(self.depth_paths) < self.n_img or len(poses) < self.n_img:
            raise RuntimeError("%s: %d colour images but %d depth images and %d poses" % (self.input_folder, self.n_img, len(self.depth_paths),
                                                                                         len(poses)))
        self.poses = []
        for p in poses[:self.n_img]:
            p = p.clone()
            p[:3, 3] *= cfg["scale"]
            self.poses.append(p)
        self._params = None

    def __len__(self):
        return self.n_img

    def _params_for(self, color, depth):
        key = (color.shape[:2], depth.shape[:2])
        if self._params is None or self._params[0] != key:
            self._params = (key, frame_params(self.cfg, color.shape, depth.shape))
        return self._params[1]

    def _stage(self, idx):
        color, depth = decode(self.color_paths[idx], self.depth_paths[idx])
        c = torch.from_numpy(np.ascontiguousarray(color)).pin_memory()
        d = torch.from_numpy(np.ascontiguousarray(depth).view(np.int16)).pin_memory()
        return idx, c, d

    def _finish(self, staged, upload):
        idx, c, d = staged
        params = self._params_for(c, d)
        with torch.cuda.stream(upload):
            cd = c.to(self.device, non_blocking=True)
            dd = d.to(self.device, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(upload)
        main = torch.cuda.current_stream(self.device)
        main.wait_event(ev)
        cd.record_stream(main)
        dd.record_stream(main)
        color, depth = prepare_frame(params, cd, dd, main)
        return idx, color, depth, self.poses[idx]

    def __getitem__(self, idx):
        upload = torch.cuda.Stream(self.device)
        return self._finish(self._stage(idx), upload)

    def __iter__(self):
        upload = torch.cuda.Stream(self.device)
        if self.prefetch <= 0:
            for idx in range(self.n_img):
                yield self._finish(self._stage(idx), upload)
            return
        q = queue.Queue(maxsize=self.prefetch)
        stop = threading.Event()

        def put(item):
            while not stop.is_set():
                try:
                    q.put(item, timeout=0.05)
                    return
                except queue.Full:
                    pass

        def work():
            try:
                for idx in range(self.n_img):
                    if stop.is_set():
                        return
                    put(self._stage(idx))
            except BaseException as e:          # handed to the consumer, which raises it
                put(e)

        t = threading.Thread(target=work, name="nsb-frame-decoder", daemon=True)
        t.start()
        try:
            for _ in range(self.n_img):
                item = q.get()
                if isinstance(item, BaseException):
                    raise item
                yield self._finish(item, upload)
        finally:
            stop.set()
            while t.is_alive():
                try:
                    q.get_nowait()
                except queue.Empty:
                    pass
                t.join(timeout=0.05)
