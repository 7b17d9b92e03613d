"""Detection on raw camera frames: the eval branch of the reference dataset's __getitem__ (kitti_dataset.py:121-163 with no
augmentation), the eval forward and the tester's decode (tester_helper.py:74-100 without the result files) behind one call.

  Detector(model, cls_mean_size, topk, threshold, resolution, max_batch, max_frame)
  Detector.from_config(cfg, checkpoint)      build_monodetr(cfg['model']) + a checkpoint in the reference's format
  detect(frames, P2)                         -> B float32 arrays (n_b, 14): [cls, alpha, x0, y0, x1, y1, h, w, l, X, Y, Z, ry, score]
  detect_device(frames, P2)                  -> (rows (B, topk, 14), count (B,) int32) on the device, no host synchronisation

`frames` is a list of (H, W, 3) uint8 RGB images (numpy arrays or torch tensors, on the host or the device; sizes may differ
within a call), `P2` the (B, 3, 4) camera matrices.  Each image is warped from its centre to `resolution` with
get_affine_transform(img_size / 2, img_size, 0, resolution, inv=1), and the forward reads calibs = P2 and img_sizes = (W, H) of
the original frames, as the reference's val loader gives them.

Graph path (per batch size, as the Trainer does it): the first call runs eagerly, which builds the lazily made state (weight
splits, split-K workspace, sine tables, reference points); the second captures pre-process + forward + extract + decode as ONE
CUDA graph, and it and every later call replay it.  At most MAX_GRAPHS batch sizes are captured, further sizes run eagerly, and
MDB_NO_GRAPH=1 turns the graphs off.  A replay reads everything from static device buffers: one staging buffer with max_batch
slots of max_frame bytes each (the frames are copied into their slots), the warp's metadata, calibs and img_sizes, all
rewritten before the replay by one pinned upload.  The weights are split inside the graph and the frozen BatchNorm fold is
refreshed in place before a replay, so a load_state_dict into the model (in place, same device) needs no new capture.
Replayed and eager calls launch the same kernels on the same inputs and give the same bits.
"""
import os

import numpy as np
import torch

from .backbone import BackboneBase
from .decode import OUT_COLS, decode_detections_device, extract_dets_from_outputs
from .labels import CLS_MEAN_SIZE
from .preprocess import ImageBatchPreprocessor, get_affine_transform, metadata_words

_ALIGN = 256


def _round_up(n):
    return (int(n) + _ALIGN - 1) // _ALIGN * _ALIGN


def _pinned(nbytes):
    """A page-locked host buffer from torch's caching host allocator, which reuses a block only after the copies that read it
    have finished."""
    return torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)


def _require_cuda(device):
    if device.type != "cuda":
        raise RuntimeError("Detector: a CUDA device is required (there is no CPU path)")


class _Silent:
    def info(self, msg):
        pass


class _Graph:
    """One captured call for one batch size and its static outputs."""

    def __init__(self):
        self.graph, self.rows, self.count = torch.cuda.CUDAGraph(), None, None


def check_inputs(frames, P2, max_frame):
    """The checks of `detect` before anything is launched: (frames as a list, P2 as a (B, 3, 4) float32 host array).
    ValueError naming the offending image."""
    if isinstance(frames, (np.ndarray, torch.Tensor)) or not hasattr(frames, "__len__"):
        raise ValueError("frames must be a list of (H, W, 3) uint8 images")
    frames = list(frames)
    for i, f in enumerate(frames):
        if not isinstance(f, (np.ndarray, torch.Tensor)):
            raise ValueError(f"frame {i}: a numpy array or torch tensor is expected, got {type(f).__name__}")
        if f.dtype != (torch.uint8 if isinstance(f, torch.Tensor) else np.uint8):
            raise ValueError(f"frame {i}: dtype {f.dtype}, uint8 is expected")
        if f.ndim != 3 or f.shape[2] != 3:
            raise ValueError(f"frame {i}: shape {tuple(f.shape)}, (H, W, 3) is expected")
        H, W = int(f.shape[0]), int(f.shape[1])
        if H < 1 or W < 1 or W > max_frame[0] or H > max_frame[1]:
            raise ValueError(f"frame {i}: {W} x {H} is empty or larger than max_frame {max_frame[0]} x {max_frame[1]}")
    if isinstance(P2, torch.Tensor):
        P2 = P2.detach().cpu().numpy()
    try:
        P2 = np.asarray(P2, dtype=np.float64)
    except (TypeError, ValueError) as e:
        raise ValueError(f"P2: not an array of numbers ({e})") from None
    if P2.ndim != 3 or P2.shape[1:] != (3, 4):
        raise ValueError(f"P2: shape {P2.shape}, (B, 3, 4) is expected")
    if P2.shape[0] != len(frames):
        raise ValueError(f"{len(frames)} frames but {P2.shape[0]} P2 matrices")
    with np.errstate(over="ignore"):                      # a value beyond float32 becomes inf and is refused below
        P2 = P2.astype(np.float32)
    for i in range(len(frames)):
        if not np.isfinite(P2[i]).all():
            raise ValueError(f"P2 of frame {i} is not finite")
    return frames, P2


class Detector:
    MAX_GRAPHS = 2

    def __init__(self, model, cls_mean_size=CLS_MEAN_SIZE, topk=50, threshold=0.2, resolution=(1280, 384), max_batch=32,
                 max_frame=(1242, 376), device="cuda"):
        self.device = torch.device(device)
        _require_cuda(self.device)
        if int(topk) < 1:
            raise ValueError(f"Detector: topk must be at least 1, got {topk}")
        if not 1 <= int(max_batch) <= 65535:
            raise ValueError(f"Detector: max_batch must be in 1..65535, got {max_batch}")
        if int(max_frame[0]) < 1 or int(max_frame[1]) < 1:
            raise ValueError(f"Detector: max_frame must be positive (W, H), got {max_frame}")
        mean = np.asarray(cls_mean_size, np.float32)
        if mean.ndim != 2 or mean.shape[1] != 3 or not np.isfinite(mean).all():
            raise ValueError("Detector: cls_mean_size must be a finite (C, 3) array")
        self.model = model.eval()
        # the backbones whose frozen BatchNorm fold a replay reads (refreshed in place before each replay)
        self._backbones = [m for m in model.modules() if isinstance(m, BackboneBase)]
        self.topk, self.threshold = int(topk), float(threshold)
        self.resolution = (int(resolution[0]), int(resolution[1]))
        self.max_batch = int(max_batch)
        self.max_frame = (int(max_frame[0]), int(max_frame[1]))
        self.preprocessor = ImageBatchPreprocessor(self.resolution, device=self.device)
        self.cls_mean_size = torch.from_numpy(mean).to(self.device)       # uploaded once: a per-call upload would be captured
        # the static staging buffer: warp metadata | calibs (f32) | img_sizes (i64) | max_batch frame slots
        mb = self.max_batch
        self._slot = _round_up(self.max_frame[0] * self.max_frame[1] * 3)
        self._calib_off = _round_up(metadata_words(mb) * 8)
        self._size_off = self._calib_off + _round_up(mb * 12 * 4)
        self._frame_off = self._size_off + _round_up(mb * 2 * 8)
        self._stage = torch.empty(self._frame_off + mb * self._slot, dtype=torch.uint8, device=self.device)
        self._calibs = self._stage[self._calib_off:self._calib_off + mb * 48].view(torch.float32).view(mb, 3, 4)
        self._sizes = self._stage[self._size_off:self._size_off + mb * 16].view(torch.int64).view(mb, 2)
        self._trans_inv = {}                  # (W, H) -> trans_inv (2, 3)
        self._graphs = {}                     # batch size -> _Graph
        self._seen = {}                       # batch size -> calls so far
        self.use_graphs = not os.environ.get("MDB_NO_GRAPH")
        self._side = torch.cuda.Stream(self.device)

    @classmethod
    def from_config(cls, cfg, checkpoint, **kwargs):
        """A Detector for `build_monodetr(cfg['model'])` with the `model_state` of `checkpoint` (the reference's format, as
        trainer.load_checkpoint reads it).  `topk` / `threshold` come from cfg['tester'] when that section is present, and
        cls_mean_size is what the reference's dataset decodes with: labels.CLS_MEAN_SIZE with cfg['dataset']['meanshape'], zeros
        without it.  Keyword arguments override any of these and pass the rest of the constructor's arguments."""
        from . import build_monodetr
        from .trainer import load_checkpoint
        device = torch.device(kwargs.get("device", "cuda"))
        model, _ = build_monodetr(cfg["model"], criterion_builder=lambda c: None)
        model = model.to(device)
        load_checkpoint(model, None, checkpoint, map_location=device, logger=_Silent())
        opts = {}
        tester = cfg.get("tester") or {}
        for key in ("topk", "threshold"):
            if key in tester:
                opts[key] = tester[key]
        meanshape = (cfg.get("dataset") or {}).get("meanshape", False)
        opts["cls_mean_size"] = CLS_MEAN_SIZE if meanshape else np.zeros_like(CLS_MEAN_SIZE, dtype=np.float32)
        opts.update(kwargs)
        return cls(model, **opts)

    @property
    def live_graphs(self):
        return len(self._graphs)

    def detect(self, frames, P2):
        """List of B float32 arrays (n_b, 14), the rows `decode_detections` gives for each frame, from one device->host copy."""
        if isinstance(frames, (list, tuple)) and len(frames) == 0:
            return []
        rows, count = self.detect_device(frames, P2)
        packed = torch.cat([rows.flatten(1), count.to(torch.float32).unsqueeze(1)], dim=1).cpu().numpy()      # the one copy
        return [packed[b, :-1].reshape(-1, OUT_COLS)[:int(packed[b, -1])].copy() for b in range(len(packed))]

    def detect_device(self, frames, P2):
        """(rows (B, topk, 14), count (B,) int32) on the device: the count[b] leading rows of frame b are its detections, the
        others zero.  Nothing waits for the device.  Calls of more than max_batch frames run in chunks of max_batch, in order."""
        frames, P2 = check_inputs(frames, P2, self.max_frame)
        if not frames:
            return (torch.zeros(0, self.topk, OUT_COLS, device=self.device),
                    torch.zeros(0, dtype=torch.int32, device=self.device))
        out = [self._chunk(frames[i:i + self.max_batch], P2[i:i + self.max_batch])
               for i in range(0, len(frames), self.max_batch)]
        if len(out) == 1:
            return out[0]
        return torch.cat([r for r, _ in out]), torch.cat([c for _, c in out])

    def trans_inv(self, W, H):
        """The eval branch's trans_inv of a W x H frame (kitti_dataset.py:129-152 without augmentation)."""
        key = (int(W), int(H))
        if key not in self._trans_inv:
            img_size = np.array(key)
            self._trans_inv[key] = get_affine_transform(img_size / 2, img_size, 0, np.array(self.resolution), inv=1)[1]
        return self._trans_inv[key]

    def _refresh_folds(self):
        for m in self._backbones:
            m._bn_tensors()

    # ---- one chunk of at most max_batch frames --------------------------------------------------------------------------------
    def _stage_inputs(self, frames, P2):
        """Copies the frames into their slots and rewrites the static metadata, calibs and img_sizes, on the current stream:
        one pinned upload, plus one device copy per CUDA frame."""
        n = len(frames)
        on_host = [not (isinstance(f, torch.Tensor) and f.is_cuda) for f in frames]
        nbytes = self._frame_off + (n * self._slot if any(on_host) else 0)
        host = _pinned(nbytes)
        h = host.numpy()
        sizes = np.array([[f.shape[1], f.shape[0]] for f in frames], np.int64)
        base = self._stage.data_ptr() + self._frame_off
        self.preprocessor.metadata(h[:self._calib_off].view(np.int64), [base + i * self._slot for i in range(n)], 3 * sizes[:, 0],
                                   sizes, np.stack([self.trans_inv(W, H) for W, H in sizes]))
        h[self._calib_off:self._calib_off + n * 48].view(np.float32)[:] = P2.reshape(-1)
        h[self._size_off:self._size_off + n * 16].view(np.int64)[:] = sizes.reshape(-1)
        for i, f in enumerate(frames):
            if on_host[i]:
                o = self._frame_off + i * self._slot
                dst = h[o:o + f.shape[0] * f.shape[1] * 3].reshape(f.shape[0], f.shape[1], 3)
                np.copyto(dst, f.numpy() if isinstance(f, torch.Tensor) else f)
        self._stage[:nbytes].copy_(host, non_blocking=True)
        for i, f in enumerate(frames):
            if not on_host[i]:
                o = self._frame_off + i * self._slot
                self._stage[o:o + f.shape[0] * f.shape[1] * 3].view(f.shape[0], f.shape[1], 3).copy_(f)

    def _forward(self, n):
        """pre-process + eval forward + extract + decode of the n staged frames: reads only static device buffers."""
        W, H = self.resolution
        inputs = torch.empty(n, 3, H, W, dtype=torch.float32, device=self.device)
        self.preprocessor.launch(self._stage.data_ptr(), n, inputs)
        calibs, img_sizes = self._calibs[:n], self._sizes[:n]
        outputs = self.model(inputs, calibs, None, img_sizes, dn_args=0)
        dets = extract_dets_from_outputs(outputs, topk=self.topk)
        return decode_detections_device(dets, img_sizes, calibs, self.cls_mean_size, self.threshold)

    def _chunk(self, frames, P2):
        n = len(frames)
        with torch.no_grad(), torch.cuda.device(self.device):
            self._stage_inputs(frames, P2)
            seen = self._seen.get(n, 0)
            self._seen[n] = seen + 1
            g = self._graphs.get(n)
            if g is None and self.use_graphs and seen >= 1 and len(self._graphs) < self.MAX_GRAPHS:
                # second call of this batch size: capture (nothing executes), then replay below
                self._refresh_folds()
                g = _Graph()
                with torch.cuda.graph(g.graph):
                    g.rows, g.count = self._forward(n)
                self._graphs[n] = g
            if g is not None:
                self._refresh_folds()
                g.graph.replay()
                return g.rows.clone(), g.count.clone()
            # first call of a batch size (or more sizes than graphs): eager, on a side stream as a capture warm-up wants it
            cur = torch.cuda.current_stream()
            self._side.wait_stream(cur)
            with torch.cuda.stream(self._side):
                rows, count = self._forward(n)
            cur.wait_stream(self._side)
            rows.record_stream(cur)
            count.record_stream(cur)
            return rows, count
