"""TEST INFRASTRUCTURE ONLY -- runs the UNMODIFIED reference Segment Anything model
(``tfimm/architectures/segment_anything/{sam,image_encoder,prompt_encoder,mask_decoder,transformer,common}.py``) on
the TensorFlow shim, as ``oracle/ref_runner.py`` does for the classifiers.

The package ``__init__`` of ``segment_anything`` is bypassed: it imports the predictor (and, through it, more of the
reference than the model needs); every module that IS imported is the reference's file.  The shim gets the TF calls
these modules make and the classifiers do not (``extend_shim``).  They are added here, at run time, rather than in
``oracle/tf_shim`` so that the classifier pins keep running on exactly the shim they were recorded with.

Restated TF semantics (TensorFlow 2.12):

* ``tf.cond(pred, true_fn, false_fn)``: eager, only the taken branch runs.
* ``tf.einsum``, ``tf.range``, ``tf.math.maximum``, ``tf.sqrt``, ``tf.sin`` / ``tf.cos``, ``tf.cumsum``,
  ``tf.broadcast_to``, ``tf.nn.relu``: elementwise / index semantics as documented.
* ``tf.image.resize(method="bilinear")`` (``antialias=False``): ResizeBilinear with ``half_pixel_centers=True``:
  source coordinate ``(o + 0.5) * in / out - 0.5``, clamped below at 0, the upper neighbour clamped to the last
  pixel.  TF returns float32; here the input's float dtype is kept, so that float64 runs of the reference stay
  float64 (in TF a float32 result cannot even be added to a float64 stream).
* ``tf.keras.layers.Conv2DTranspose(k, strides=s, padding="valid")``: kernel ``(kh, kw, out, in)``, output
  ``(in - 1) * s + k``.
"""
import types

import torch
import torch.nn.functional as F

from . import ref_runner as rr

_MODULES = ("common", "image_encoder", "prompt_encoder", "transformer", "mask_decoder", "sam")


def _bilinear_weights(n_in, n_out):
    src = ((torch.arange(n_out, dtype=torch.float64) + 0.5) * (n_in / n_out) - 0.5).clamp(min=0.0)
    lo = src.floor().long().clamp(max=n_in - 1)
    hi = (lo + 1).clamp(max=n_in - 1)
    frac = src - lo.double()
    m = torch.zeros(n_out, n_in, dtype=torch.float64)
    m[torch.arange(n_out), lo] += 1.0 - frac
    m[torch.arange(n_out), hi] += frac
    return m


def extend_shim(tf):
    """Adds the TF calls of the Segment Anything modules to the shim module ``tf`` (idempotent)."""
    if tf.__dict__.get("_sam_extended"):   # the shim answers every unknown attribute, so look in its namespace
        return
    T, _t = tf.Tensor, tf._t

    def cond(pred, true_fn=None, false_fn=None, name=None):
        return true_fn() if bool(pred) else false_fn()

    def einsum(equation, *inputs, **_):
        return torch.einsum(equation, *[_t(x).as_subclass(torch.Tensor) for x in inputs]).as_subclass(T)

    def range_(start, limit=None, delta=1, dtype=None, name=None):
        if limit is None:
            start, limit = 0, start
        return torch.arange(int(start), int(limit), int(delta), dtype=tf._dtype(dtype) if dtype else torch.int32
                            ).as_subclass(T)

    def maximum(x, y, name=None):
        if not isinstance(x, torch.Tensor) and not isinstance(y, torch.Tensor):
            return _t(max(x, y))
        return torch.maximum(_t(x), _t(y))

    def cumsum(x, axis=0, **_):
        return torch.cumsum(_t(x), dim=axis)

    def broadcast_to(input, shape, name=None):  # noqa: A002
        return _t(input).expand(*[int(s) for s in shape]).clone()

    resize_other = tf.image.resize

    def resize(images, size, method="bilinear", **kw):
        if method != "bilinear":
            return resize_other(images, size, method=method, **kw)
        x = _t(images)
        squeeze = x.dim() == 3
        if squeeze:
            x = x[None]
        dt = x.dtype if x.is_floating_point() else torch.float32
        mh = _bilinear_weights(x.shape[1], int(size[0]))
        mw = _bilinear_weights(x.shape[2], int(size[1]))
        y = torch.einsum("oh,bhwc->bowc", mh, x.as_subclass(torch.Tensor).to(torch.float64))
        y = torch.einsum("pw,bowc->bopc", mw, y).to(dt)
        return (y[0] if squeeze else y).as_subclass(T)

    class Conv2DTranspose(tf.keras.layers.Conv2D):
        def build(self, input_shape):
            cin = input_shape[-1]
            self.kernel = self.add_weight("kernel", (*self.kernel_size, self.filters, cin),
                                          initializer=self.kernel_initializer)
            self.bias = self.add_weight("bias", (self.filters,), initializer=self.bias_initializer) if self.use_bias \
                else None

        def call(self, x):
            assert self.padding.lower() == "valid"
            w = self.kernel.as_subclass(torch.Tensor).permute(3, 2, 0, 1).to(x.dtype)
            y = F.conv_transpose2d(x.as_subclass(torch.Tensor).permute(0, 3, 1, 2), w, None, stride=self.strides)
            y = y.permute(0, 2, 3, 1).as_subclass(T)
            if self.bias is not None:
                y = y + self.bias
            return self.activation(y)

    tf.cond, tf.einsum, tf.range, tf.cumsum, tf.broadcast_to = cond, einsum, range_, cumsum, broadcast_to
    tf.sqrt = lambda x: torch.sqrt(_t(x))
    tf.sin = lambda x: torch.sin(_t(x))
    tf.cos = lambda x: torch.cos(_t(x))
    tf.math.maximum = maximum
    tf.nn.relu = lambda x: torch.relu(_t(x))
    tf.image.resize = resize
    tf.image.ResizeMethod = types.SimpleNamespace(BILINEAR="bilinear", BICUBIC="bicubic")
    tf.keras.layers.Conv2DTranspose = Conv2DTranspose
    tf._sam_extended = True


def _import_sam():
    import importlib
    import sys

    import tensorflow as tf

    extend_shim(tf)
    mods = rr._import_reference()
    pkg_name = "tfimm.architectures.segment_anything"
    if pkg_name not in sys.modules:
        pkg = types.ModuleType(pkg_name)
        pkg.__path__ = [str(rr.REFERENCE / "tfimm" / "architectures" / "segment_anything")]
        sys.modules[pkg_name] = pkg
    for m in _MODULES:
        mods[m] = importlib.import_module(f"{pkg_name}.{m}")
    return mods


class ReferenceSAM(rr.ReferenceModel):
    """A reference ``SegmentAnythingModel`` built by the reference's ``create_model`` on the shim.  Its variables
    exist once ``build()`` has called the whole model once on its ``dummy_inputs`` (Keras builds lazily)."""

    def build(self):
        with rr._reference_modules(), torch.no_grad():
            self.model(self.model.dummy_inputs, training=False)
        return self

    def image_encoder(self, x, return_features=False):
        with rr._reference_modules(), torch.no_grad():
            out = self.model.image_encoder(x.detach().cpu().numpy(), training=False, return_features=return_features)
        conv = lambda t: t.as_subclass(torch.Tensor).detach().clone()  # noqa: E731
        if return_features:
            return conv(out[0]), {k: conv(v) for k, v in out[1].items()}
        return conv(out)


def create_model(model_name: str, **kwargs) -> ReferenceSAM:
    with rr._reference_modules():
        mods = _import_sam()
        model = mods["factory"].create_model(model_name, **kwargs)
    return ReferenceSAM(model, mods)


# the reference's own test configuration, tests/models/test_segment_anything.py:55-72 of the reference
TEST_MODEL_FIELDS = dict(name="sam_vit_test_model", input_size=(32, 32), fixed_input_size=False, embed_dim=12,
                         encoder_patch_size=4, encoder_embed_dim=12, encoder_nb_blocks=3, encoder_nb_heads=2,
                         encoder_global_attn_indices=(1,), encoder_window_size=2, decoder_nb_heads=2,
                         decoder_mlp_channels=14, decoder_iou_hidden_dim=18)


def register_test_model(**cfg_fields):
    """Registers a model in the reference's registry with the fields of ``TEST_MODEL_FIELDS``, overridden by
    ``cfg_fields`` (``name`` included)."""
    with rr._reference_modules():
        mods = _import_sam()
        sam = mods["sam"]
        fields = {**TEST_MODEL_FIELDS, **cfg_fields}

        def sam_vit_test_model():
            return sam.SegmentAnythingModel, sam.SegmentAnythingModelConfig(**fields)

        sam_vit_test_model.__name__ = fields["name"]
        mods["registry"].register_model(sam_vit_test_model)


def model_config(model_name: str):
    import dataclasses

    with rr._reference_modules():
        mods = _import_sam()
        return dataclasses.asdict(mods["registry"].model_config(model_name))


def list_models(module: str = "sam"):
    with rr._reference_modules():
        mods = _import_sam()
        return mods["registry"].list_models(module=module)
