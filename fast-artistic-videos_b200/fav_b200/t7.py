"""Torch7 `.t7` checkpoint reader (SURVEY.md §8 f-1): lets `checkpoint-*-video.t7` files of the reference load.

`torch.load(path).model` is the only way weights enter the reference (fast_artistic_video_core.lua:38-47); the checkpoint
table is `{opt, ..., iter, model}` with the model a float `nn.Sequential` (train_video.lua:507-541).

The serialisation format lives in the un-vendored torch7 rock (`File.lua`): PARITY UNPINNED.  It is restated here from
its published description (binary mode, little endian, 8-byte longs):
  object := int32 type, then
    0 nil | 1 number: float64 | 2 string: int32 len + bytes | 5 boolean: int32
    3 table : int32 index, [int32 count, count x (key object, value object)]   (index seen before => back-reference)
    4 torch : int32 index, [string "V <n>", string className, payload]          (same back-reference rule)
       tensor payload : int32 ndim, int64 size[ndim], int64 stride[ndim], int64 storageOffset (1-based), storage object
       storage payload: int64 n, n raw elements
       any other class: one table object holding its fields (nn modules have no custom :write)
`write_checkpoint` produces files in the same format from a state dict (used by the tests; there is no network to fetch
the released checkpoints, so the reader is validated on round trips only).
"""
from __future__ import annotations

import struct
from typing import Dict, List, Tuple

import numpy as np

TYPE_NIL, TYPE_NUMBER, TYPE_STRING, TYPE_TABLE, TYPE_TORCH, TYPE_BOOLEAN = 0, 1, 2, 3, 4, 5

_TENSOR = {"torch.FloatTensor": np.float32, "torch.DoubleTensor": np.float64, "torch.LongTensor": np.int64,
           "torch.IntTensor": np.int32, "torch.ByteTensor": np.uint8, "torch.CudaTensor": np.float32}
_STORAGE = {k.replace("Tensor", "Storage"): v for k, v in _TENSOR.items()}


class T7Object(dict):
    """A deserialised torch class instance: dict of fields + .torch_type."""

    def __init__(self, torch_type, fields=None):
        super().__init__(fields or {})
        self.torch_type = torch_type


class _Reader:
    def __init__(self, data: bytes):
        self.d, self.p, self.objects = data, 0, {}

    def _unpack(self, fmt, n):
        v = struct.unpack_from("<" + fmt, self.d, self.p)
        self.p += n
        return v[0]

    def int(self):
        return self._unpack("i", 4)

    def long(self):
        return self._unpack("q", 8)

    def string(self):
        n = self.int()
        s = self.d[self.p:self.p + n].decode("latin1")
        self.p += n
        return s

    def obj(self):
        t = self.int()
        if t == TYPE_NIL:
            return None
        if t == TYPE_NUMBER:
            return self._unpack("d", 8)
        if t == TYPE_STRING:
            return self.string()
        if t == TYPE_BOOLEAN:
            return self.int() == 1
        if t == TYPE_TABLE:
            idx = self.int()
            if idx in self.objects:
                return self.objects[idx]
            tab = {}
            self.objects[idx] = tab
            for _ in range(self.int()):
                k = self.obj()
                v = self.obj()
                if isinstance(k, float) and k == int(k):
                    k = int(k)
                tab[k] = v
            return tab
        if t == TYPE_TORCH:
            idx = self.int()
            if idx in self.objects:
                return self.objects[idx]
            version = self.string()
            cls = self.string() if version.startswith("V ") else version  # legacy files have no version string
            if cls in _TENSOR:
                nd = self.int()
                size = [self.long() for _ in range(nd)]
                stride = [self.long() for _ in range(nd)]
                off = self.long() - 1
                self.objects[idx] = None
                storage = self.obj()
                if storage is None or nd == 0:
                    arr = np.zeros(size or (0,), _TENSOR[cls])
                else:
                    arr = np.lib.stride_tricks.as_strided(storage[off:], shape=size,
                                                          strides=[s * storage.itemsize for s in stride]).copy()
                self.objects[idx] = arr
                return arr
            if cls in _STORAGE:
                n = self.long()
                dt = np.dtype(_STORAGE[cls]).newbyteorder("<")
                arr = np.frombuffer(self.d, dt, count=n, offset=self.p).copy()
                self.p += n * dt.itemsize
                self.objects[idx] = arr
                return arr
            o = T7Object(cls)
            self.objects[idx] = o
            fields = self.obj()
            if isinstance(fields, dict):
                o.update(fields)
            return o
        raise ValueError(f".t7: unsupported object type {t} at byte {self.p}")


def load(path: str):
    with open(path, "rb") as f:
        return _Reader(f.read()).obj()


# ---- nn.Sequential -> (arch string, state dict in fav.h naming) ------------------------------------------------------
def _cls(m):
    return m.torch_type.split(".", 1)[1] if isinstance(m, T7Object) else None


def _mods(m) -> List:
    mods = m.get("modules", {})
    return [mods[k] for k in sorted(mods)]


NORMS = ("InstanceNormalization", "SpatialBatchNormalization")  # nn.* / cudnn.* classes alike (_cls drops the package)


class GeometryError(ValueError):
    """The checkpoint's module tree does not have the geometry build_model would give its arch string."""


def model_to_state(model, geometry: dict = None) -> Tuple[str, Dict[str, np.ndarray], float, int]:
    """Walk the checkpoint's nn.Sequential exactly as models_video.build_model lays it out (models_video.lua:55-140,
    plus the lazily inserted SpatialReflectionPadding, train_video.lua:319-324) and return
    (arch string, {name: array}, tanh_constant, reflect_pad).  `geometry`, if given, receives what the file says about
    padding: 'padding_type' ('reflect-start' | 'zero', inferred from the residual blocks: pad-0 convs + ShaveImage vs pad-1
    convs + Identity, models_video.lua:21-53), 'has_reflect_pad', and every conv's (name, padW, padW implied by its token);
    a layout build_model cannot produce for these two padding types raises GeometryError instead of being run with a
    different geometry.  geometry['norm'] is 'instance' (InstanceNormalization) or 'batch' (nn. / cudnn.SpatialBatchNormalization,
    -use_instance_norm 0, models_video.lua:21-25,33-37,121-127: weight / bias, nil when affine = false, are read as 1 / 0, plus
    running_mean, running_var and eps); a checkpoint mixing the two, a BatchNorm without running statistics or one whose size
    is not its convolution's output channel count raises GeometryError."""
    toks, state, tanh_c, pad = [], {}, 150.0, 0
    geo = geometry if geometry is not None else {}
    geo.update(padding_type=None, has_reflect_pad=False, conv_pads=[], norm=None)
    chan = None  # output channels of the last convolution

    def check_pad(name, m, implied):
        pw, ph = int(m.get("padW", 0)), int(m.get("padH", m.get("padW", 0)))
        geo["conv_pads"].append((name, pw, implied))
        if pw != implied or ph != implied:
            raise GeometryError(f".t7 model: {name} has padding {pw}x{ph}, its arch token implies {implied}")
    mods = _mods(model)
    i = 0

    def conv_params(name, m, transposed):
        nonlocal chan
        w = np.asarray(m["weight"], np.float32)
        cin, cout, k = int(m["nInputPlane"]), int(m["nOutputPlane"]), int(m["kW"])
        chan = cout
        state[name + ".weight"] = w.reshape((cin, cout, k, k) if transposed else (cout, cin, k, k))
        state[name + ".bias"] = np.asarray(m["bias"], np.float32).reshape(cout)

    def in_params(name, m):
        kind = "batch" if _cls(m) == "SpatialBatchNormalization" else "instance"
        if geo["norm"] not in (None, kind):
            raise GeometryError(f".t7 model: {name} is a {m.torch_type} after {geo['norm']} normalisation layers; a checkpoint "
                                "uses one normalisation type throughout (-use_instance_norm, train_video.lua:22)")
        geo["norm"] = kind
        if kind == "instance":
            state[name + ".weight"] = np.asarray(m["weight"], np.float32).reshape(-1)
            state[name + ".bias"] = np.asarray(m["bias"], np.float32).reshape(-1)
            return
        for f in ("running_mean", "running_var"):  # evaluate mode normalises with the running statistics
            if m.get(f) is None:
                raise GeometryError(f".t7 model: {name} ({m.torch_type}) has no {f}")
        mean = np.asarray(m["running_mean"], np.float32).reshape(-1)
        var = np.asarray(m["running_var"], np.float32).reshape(-1)
        if not mean.size == var.size == chan:
            raise GeometryError(f".t7 model: {name} ({m.torch_type}) has {var.size} channels, its convolution {chan}")
        w, b = m.get("weight"), m.get("bias")  # nil when affine = false
        state[name + ".weight"] = np.ones(chan, np.float32) if w is None else np.asarray(w, np.float32).reshape(-1)
        state[name + ".bias"] = np.zeros(chan, np.float32) if b is None else np.asarray(b, np.float32).reshape(-1)
        if not state[name + ".weight"].size == state[name + ".bias"].size == chan:
            raise GeometryError(f".t7 model: {name} ({m.torch_type}) weight / bias do not have {chan} channels")
        state[name + ".running_mean"], state[name + ".running_var"] = mean, var
        state[name + ".eps"] = np.full(1, m.get("eps", 1e-5), np.float32)

    def take_norm_relu(name):
        nonlocal i
        if i < len(mods) and _cls(mods[i]) in NORMS:
            in_params(name + ".n", mods[i])
            i += 1
        if i < len(mods) and _cls(mods[i]) == "ReLU":
            i += 1

    while i < len(mods):
        m = mods[i]
        c = _cls(m)
        name = f"l{len(toks)}"
        i += 1
        if c == "SpatialReflectionPadding":
            pad = int(m["pad_l"])
            if not (i == 1 and pad == int(m["pad_r"]) == int(m["pad_t"]) == int(m["pad_b"])):
                raise GeometryError(".t7 model: only the leading symmetric SpatialReflectionPadding of padding_type "
                                    "'reflect-start' is supported (train_video.lua:319-324)")
            geo["has_reflect_pad"] = True
        elif c == "SpatialConvolution":
            k, s = int(m["kW"]), int(m["dW"])
            if k == 3 and s == 2 and int(m["padW"]) == 1:
                toks.append(f"d{int(m['nOutputPlane'])}")
            else:
                toks.append(f"c{k}s{s}-{int(m['nOutputPlane'])}")
            check_pad(name, m, 1 if toks[-1][0] == "d" else (k - 1) // 2)  # models_video.lua:65-80,90-93
            conv_params(name, m, False)
            take_norm_relu(name)
        elif c == "SpatialFullConvolution":
            k, s = int(m["kW"]), int(m["dW"])
            toks.append(f"u{int(m['nOutputPlane'])}" if (k == 3 and s == 2) else f"f{k}s{s}-{int(m['nOutputPlane'])}")
            check_pad(name, m, (k - 1) // 2)  # :81-89,99-102
            conv_params(name, m, True)
            take_norm_relu(name)
        elif c == "SpatialUpSamplingNearest":
            toks.append(f"U{int(m['scale_factor'])}")
            take_norm_relu(name)
        elif c == "Sequential":  # residual block: Sequential{ConcatTable{conv_block, ShaveImage}, CAddTable}
            concat = _mods(m)[0]
            block = _mods(_mods(concat)[0])
            convs = [b for b in block if _cls(b) == "SpatialConvolution"]
            norms = [b for b in block if _cls(b) in NORMS]
            assert len(convs) == 2 and len(norms) == 2, "unexpected residual block layout"
            extra = [_cls(b) for b in block if _cls(b) not in ("SpatialConvolution", "ReLU") + NORMS]
            skip = _cls(_mods(concat)[1]) if len(_mods(concat)) > 1 else None
            rp = int(convs[0].get("padW", 0))
            ptype = "reflect-start" if (rp == 0 and skip == "ShaveImage") else ("zero" if (rp == 1 and skip == "Identity") else None)
            if extra or ptype is None or (geo["padding_type"] not in (None, ptype)):
                raise GeometryError(f".t7 model: residual block {name} (conv padding {rp}, skip {skip}, extra modules {extra}) is not "
                                    "a padding_type 'reflect-start' or 'zero' block (models_video.lua:21-53)")
            geo["padding_type"] = ptype
            for cn, cm in ((name + ".c1", convs[0]), (name + ".c2", convs[1])):
                check_pad(cn, cm, rp)
            toks.append(f"R{int(convs[0]['nOutputPlane'])}")
            conv_params(name + ".c1", convs[0], False); in_params(name + ".n1", norms[0])
            conv_params(name + ".c2", convs[1], False); in_params(name + ".n2", norms[1])
        elif c == "Tanh":
            pass
        elif c == "MulConstant":
            tanh_c = float(m["constant_scalar"])
        elif c == "TotalVariation":
            pass  # identity in forward (TotalVariation.lua:12-15)
        else:
            raise ValueError(f".t7 model: unsupported module {m.torch_type}")
    if geo["norm"] is None:
        geo["norm"] = "instance"
    if geo["padding_type"] is None:
        geo["padding_type"] = "reflect-start" if geo["has_reflect_pad"] else "zero"
    if geo["has_reflect_pad"] != (geo["padding_type"] == "reflect-start" and pad > 0) and any(t[0] in "RC" for t in toks):
        raise GeometryError(".t7 model: the leading SpatialReflectionPadding and the residual blocks' padding disagree")
    return ",".join(toks), state, tanh_c, pad


def load_checkpoint(path: str, geometry: dict = None):
    ck = load(path)
    model = ck["model"] if isinstance(ck, dict) and "model" in ck else ck
    return model_to_state(model, geometry)


# ---- writer (tests) ---------------------------------------------------------------------------------------------------
class _Writer:
    def __init__(self):
        self.b, self.n = bytearray(), 0

    def int(self, v):
        self.b += struct.pack("<i", v)

    def long(self, v):
        self.b += struct.pack("<q", v)

    def string(self, s):
        self.int(len(s))
        self.b += s.encode("latin1")

    def obj(self, o):
        if o is None:
            self.int(TYPE_NIL)
        elif isinstance(o, bool):
            self.int(TYPE_BOOLEAN); self.int(1 if o else 0)
        elif isinstance(o, (int, float)):
            self.int(TYPE_NUMBER); self.b += struct.pack("<d", float(o))
        elif isinstance(o, str):
            self.int(TYPE_STRING); self.string(o)
        elif isinstance(o, np.ndarray):
            a = np.ascontiguousarray(o, np.float32)
            self.int(TYPE_TORCH); self.n += 1; self.int(self.n); self.string("V 1"); self.string("torch.FloatTensor")
            self.int(a.ndim)
            for s in a.shape:
                self.long(s)
            st = [int(x // a.itemsize) for x in a.strides]
            for s in st:
                self.long(s)
            self.long(1)
            self.int(TYPE_TORCH); self.n += 1; self.int(self.n); self.string("V 1"); self.string("torch.FloatStorage")
            self.long(a.size)
            self.b += a.tobytes()
        elif isinstance(o, T7Object):
            self.int(TYPE_TORCH); self.n += 1; self.int(self.n); self.string("V 1"); self.string(o.torch_type)
            self.obj(dict(o))
        elif isinstance(o, dict):
            self.int(TYPE_TABLE); self.n += 1; self.int(self.n); self.int(len(o))
            for k, v in o.items():
                self.obj(k); self.obj(v)
        else:
            raise TypeError(type(o))


def write_checkpoint(path: str, arch: str, state: Dict[str, np.ndarray], tanh_constant: float = 150.0,
                     reflect_pad: int = 40, padding_type: str = "reflect-start", norm: str = "instance",
                     bn_class: str = "nn.SpatialBatchNormalization", affine: bool = True) -> None:
    """Serialise a state dict as the `{model = nn.Sequential{...}}` table train_video.lua:507-541 saves
    (padding_type 'reflect-start': leading reflection pad, pad-0 residual convs + ShaveImage; 'zero': pad-1 residual convs +
    Identity, models_video.lua:21-53).  norm='batch': `bn_class` modules (nn. or cudnn.SpatialBatchNormalization) with the
    state's running_mean / running_var / eps, in evaluate mode; affine=False leaves weight and bias nil."""
    from . import synth

    def seq(mods, cls="nn.Sequential"):
        return T7Object(cls, {"modules": {i + 1: m for i, m in enumerate(mods)}})

    def conv(name, cin, cout, k, s, p, tr=False):
        return T7Object("nn.SpatialFullConvolution" if tr else "nn.SpatialConvolution",
                        {"nInputPlane": cin, "nOutputPlane": cout, "kW": k, "kH": k, "dW": s, "dH": s, "padW": p, "padH": p,
                         "weight": state[name + ".weight"], "bias": state[name + ".bias"]})

    def inorm(name):
        if norm == "batch":
            f = {"running_mean": state[name + ".running_mean"], "running_var": state[name + ".running_var"],
                 "eps": float(state[name + ".eps"].reshape(-1)[0]), "momentum": 0.1, "affine": affine, "train": False}
            if affine:
                f.update(weight=state[name + ".weight"], bias=state[name + ".bias"])
            return T7Object(bn_class, f)
        return T7Object("nn.InstanceNormalization", {"weight": state[name + ".weight"], "bias": state[name + ".bias"],
                                                      "eps": 1e-5, "nOutput": int(state[name + ".weight"].size)})

    zero = padding_type == "zero"
    mods = [] if zero else [T7Object("nn.SpatialReflectionPadding", {"pad_l": reflect_pad, "pad_r": reflect_pad, "pad_t": reflect_pad,
                                                                     "pad_b": reflect_pad})]
    for i, s in enumerate(synth.parse_arch(arch)):
        n = f"l{i}"
        if s["kind"] == "conv":
            mods.append(conv(n, s["cin"], s["cout"], s["k"], s["stride"], s["pad"]))
        elif s["kind"] == "fullconv":
            mods.append(conv(n, s["cin"], s["cout"], s["k"], s["stride"], s["pad"], True))
        elif s["kind"] == "up":
            mods.append(T7Object("nn.SpatialUpSamplingNearest", {"scale_factor": s["scale"]}))
        elif s["kind"] == "res":
            rp = 1 if zero else 0
            block = seq([conv(n + ".c1", s["cin"], s["cout"], 3, 1, rp), inorm(n + ".n1"), T7Object("nn.ReLU", {"inplace": True}),
                         conv(n + ".c2", s["cout"], s["cout"], 3, 1, rp), inorm(n + ".n2")])
            skip = T7Object("nn.Identity", {}) if zero else T7Object("nn.ShaveImage", {"size": 2})
            mods.append(seq([seq([block, skip], "nn.ConcatTable"), T7Object("nn.CAddTable", {})]))
        if s["in_norm"]:
            mods.append(inorm(n + ".n"))
        if s["relu"]:
            mods.append(T7Object("nn.ReLU", {"inplace": True}))
    mods += [T7Object("nn.Tanh", {}), T7Object("nn.MulConstant", {"constant_scalar": tanh_constant}),
             T7Object("nn.TotalVariation", {"strength": 1e-6})]
    w = _Writer()
    opt = {"arch": arch, "padding_type": padding_type}
    if norm == "batch":
        opt["use_instance_norm"] = 0
    w.obj({"opt": opt, "iter": 60000, "model": seq(mods)})
    with open(path, "wb") as f:
        f.write(bytes(w.b))


# ---- loss network (-evaluate, -loss_network) ---------------------------------------------------------------------------
# An nn.Sequential of SpatialConvolution[MM] / ReLU / SpatialMaxPooling (the nn.* or cudnn.* classes), as loadcaffe writes
# VGG-16 (models/vgg16.t7, fast_artistic_video.lua:63).  PerceptualCriterion trims every module after the deepest loss layer
# (layer_utils.lua:146-165), whatever its type, so VGG's classifier (View / Linear / Dropout / SoftMax) is never read.
LOSS_MODULES = ("SpatialConvolution", "SpatialConvolutionMM", "ReLU", "SpatialMaxPooling")


def _unsupported(msg):
    from . import _lib

    return _lib.FavError(_lib.FAV_ERR_UNSUPPORTED, msg)


def loss_network_from_model(model, last_index: int) -> List[dict]:
    """The first `last_index` top-level modules of a loss network as dicts: {'type': 'conv', cin, cout, k, stride, pad,
    weight [cout,cin,k,k], bias}, {'type': 'relu'}, {'type': 'pool', kW, kH, dW, dH, padW, padH, ceil_mode}.  Any other module
    before that index, and a convolution the tensor-core planner cannot run, raise FavError(FAV_ERR_UNSUPPORTED) naming the
    module and its (1-based) index."""
    mods = _mods(model)
    if last_index > len(mods):
        from . import _lib

        raise _lib.FavError(_lib.FAV_ERR_INVALID, f"loss network: layer {last_index} requested, the network has {len(mods)} modules")
    out = []
    for i, m in enumerate(mods[:last_index], 1):
        c = _cls(m)
        name = m.torch_type if isinstance(m, T7Object) else type(m).__name__
        if c not in LOSS_MODULES:
            raise _unsupported(f"loss network module {i} ({name}): only SpatialConvolution, ReLU and SpatialMaxPooling are supported "
                               "before the deepest loss layer")
        if c.startswith("SpatialConvolution"):
            cin, cout = int(m["nInputPlane"]), int(m["nOutputPlane"])
            kw, kh, dw, dh = int(m["kW"]), int(m["kH"]), int(m["dW"]), int(m["dH"])
            pw, ph = int(m.get("padW", 0)), int(m.get("padH", m.get("padW", 0)))
            ok = (kw == kh and dw == dh and pw == ph and kw % 2 == 1 and pw <= kw // 2 and (cin <= 8 or cin % 16 == 0)
                  and (dw == 1 or (dw == 2 and kw == 3 and pw == 1)) and m.get("groups", 1) in (1, None))
            if not ok:
                raise _unsupported(f"loss network module {i} ({name} {cin}->{cout}, kernel {kw}x{kh}, stride {dw}x{dh}, pad {pw}x{ph}): "
                                   "not a convolution geometry the tensor-core planner runs")
            w = np.asarray(m["weight"], np.float32).reshape(cout, cin, kw, kw)  # SpatialConvolutionMM stores [cout, cin*k*k]
            out.append(dict(type="conv", cin=cin, cout=cout, k=kw, stride=dw, pad=pw, weight=np.ascontiguousarray(w),
                            bias=np.asarray(m["bias"], np.float32).reshape(cout)))
        elif c == "ReLU":
            out.append(dict(type="relu"))
        else:
            out.append(dict(type="pool", kW=int(m["kW"]), kH=int(m["kH"]), dW=int(m["dW"]), dH=int(m["dH"]),
                            padW=int(m.get("padW", 0)), padH=int(m.get("padH", 0)), ceil_mode=bool(m.get("ceil_mode", False))))
    return out


def load_loss_network(path: str, last_index: int) -> List[dict]:
    """torch.load(opt.loss_network) (fast_artistic_video_core.lua:82), trimmed after module `last_index`."""
    return loss_network_from_model(load(path), last_index)


def write_loss_network(path: str, modules: List[dict], classifier: bool = True, cudnn: bool = False, conv_mm: bool = False) -> None:
    """Serialise a loss network (the dicts of loss_network_from_model) as an nn.Sequential .t7 file.  classifier=True appends
    VGG-16's head as loadcaffe names it (View, Linear, ReLU, Dropout, ..., SoftMax); trimming never reads it, so its Linear
    modules carry 1x1 stand-in tensors instead of the 0.5 GB of real fc weights.  cudnn=True writes the cudnn.* classes,
    conv_mm=True SpatialConvolutionMM with 2-D [cout, cin*k*k] weights."""
    pre = "cudnn." if cudnn else "nn."
    seq = []
    for m in modules:
        if m["type"] == "conv":
            k = m["k"]
            w = np.asarray(m["weight"], np.float32)
            cls = "nn.SpatialConvolutionMM" if conv_mm else pre + "SpatialConvolution"
            seq.append(T7Object(cls, {"nInputPlane": m["cin"], "nOutputPlane": m["cout"], "kW": k, "kH": k, "dW": m["stride"],
                                      "dH": m["stride"], "padW": m["pad"], "padH": m["pad"],
                                      "weight": w.reshape(m["cout"], -1) if conv_mm else w, "bias": np.asarray(m["bias"], np.float32)}))
        elif m["type"] == "relu":
            seq.append(T7Object(pre + "ReLU", {"inplace": True}))
        else:
            seq.append(T7Object(pre + "SpatialMaxPooling", {"kW": m["kW"], "kH": m["kH"], "dW": m["dW"], "dH": m["dH"],
                                                            "padW": m["padW"], "padH": m["padH"], "ceil_mode": bool(m["ceil_mode"])}))
    if classifier:
        stand_in = lambda: {"weight": np.zeros((1, 1), np.float32), "bias": np.zeros((1,), np.float32)}
        seq += [T7Object("nn.View", {"size": 25088}), T7Object("nn.Linear", stand_in()), T7Object("nn.ReLU", {"inplace": True}),
                T7Object("nn.Dropout", {"p": 0.5}), T7Object("nn.Linear", stand_in()), T7Object("nn.ReLU", {"inplace": True}),
                T7Object("nn.Dropout", {"p": 0.5}), T7Object("nn.Linear", stand_in()), T7Object("nn.SoftMax", {})]
    w = _Writer()
    w.obj(T7Object("nn.Sequential", {"modules": {i + 1: m for i, m in enumerate(seq)}}))
    with open(path, "wb") as f:
        f.write(bytes(w.b))
