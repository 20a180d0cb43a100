"""Loss layers + Accuracy.

reference: include/caffe/loss_layers.hpp:23 (Accuracy), :98 (Loss base), :153
(Contrastive), :244 (Euclidean), :355 (Hinge), :433 (Infogain), :528 (MultinomialLogistic),
:606 (SigmoidCrossEntropy), :707 (SoftmaxWithLoss); loss_layer.cpp:14-21 (default
loss_weight 1 on the first top).
"""
from __future__ import annotations


import torch

from .. import ops
from .. import proto as P
from .base import Layer, register


class LossLayer(Layer):
    exact_bottoms = 2
    exact_tops = 1
    is_loss = True

    def setup(self, bottom_shapes):
        if bottom_shapes[0][0] != bottom_shapes[1][0]:
            raise ValueError("The data and label should have the same number.")
        self.configure(bottom_shapes)
        return [(1, 1, 1, 1)]

    def configure(self, bottom_shapes):
        pass

    def allow_force_backward(self, bottom: int) -> bool:
        """The label (bottom 1) is never forced.  reference: include/caffe/loss_layers.hpp:123-125."""
        return bottom != 1


@register("SOFTMAX_LOSS")
class SoftmaxWithLossLayer(LossLayer):
    """Fused softmax + multinomial logistic loss; optional 2nd top = probabilities.
    (The reference's GPU path falls back to the CPU every iteration; ours stays on-device.)
    reference: src/caffe/layers/softmax_loss_layer.cpp:38-87, softmax_loss_layer.cu:11-22."""
    exact_tops = None
    min_tops = 1
    max_tops = 2

    def setup(self, bottom_shapes):
        super().setup(bottom_shapes)
        return [(1, 1, 1, 1), tuple(bottom_shapes[0])]

    def forward(self, x, label):
        k = ops.get(self.ctx)
        if self.n_tops == 2:
            loss, prob = k.softmax_loss(x, label, return_prob=True)
            return loss, prob
        return (k.softmax_loss(x, label),)


@register("EUCLIDEAN_LOSS")
class EuclideanLossLayer(LossLayer):
    """reference: src/caffe/layers/euclidean_loss_layer.cpp:30-46."""

    def allow_force_backward(self, bottom: int) -> bool:
        """Both bottoms may be computed blobs.  reference: include/caffe/loss_layers.hpp:259-261."""
        return True

    def forward(self, a, b):
        return (ops.reference.euclidean_loss(a, b.reshape(a.shape)),)


@register("HINGE_LOSS")
class HingeLossLayer(LossLayer):
    """reference: src/caffe/layers/hinge_loss_layer.cpp:33-67."""

    def configure(self, bottom_shapes):
        self.norm = self.lp.hinge_loss_param.enum_name("norm")

    def forward(self, x, label):
        return (ops.reference.hinge_loss(x, label, self.norm),)


@register("SIGMOID_CROSS_ENTROPY_LOSS")
class SigmoidCrossEntropyLossLayer(LossLayer):
    """reference: src/caffe/layers/sigmoid_cross_entropy_loss_layer.cpp:47-52."""

    def forward(self, x, t):
        return (ops.reference.sigmoid_cross_entropy_loss(x, t),)


@register("MULTINOMIAL_LOGISTIC_LOSS")
class MultinomialLogisticLossLayer(LossLayer):
    """reference: src/caffe/layers/multinomial_logistic_loss_layer.cpp:29-36."""

    def forward(self, prob, label):
        return (ops.reference.multinomial_logistic_loss(prob, label),)


@register("INFOGAIN_LOSS")
class InfogainLossLayer(LossLayer):
    """H comes from a BlobProto file (infogain_loss_param.source) or a 3rd bottom.
    reference: src/caffe/layers/infogain_loss_layer.cpp:14-73."""
    exact_bottoms = None
    min_bottoms = 2

    def configure(self, bottom_shapes):
        self.H = None
        if len(bottom_shapes) < 3:
            src = self.lp.infogain_loss_param.source
            if not src:
                raise ValueError("infogain matrix needs a source file or a third bottom")
            from ..utils.paths import resolve
            path = resolve(src, self.ctx.model_dir)
            blob = P.read_binary(path, P.BlobProto)
            self.H = torch.from_numpy(P.blob_to_array(blob).reshape(blob.height, blob.width).copy())

    def forward(self, prob, label, H=None):
        H = H.reshape(H.shape[-2], H.shape[-1]) if H is not None else self.H
        return (ops.reference.infogain_loss(prob, label, H),)


@register("CONTRASTIVE_LOSS")
class ContrastiveLossLayer(LossLayer):
    """reference: src/caffe/layers/contrastive_loss_layer.cpp:14-58."""
    exact_bottoms = 3

    def configure(self, bottom_shapes):
        self.margin = float(self.lp.contrastive_loss_param.margin)

    def allow_force_backward(self, bottom: int) -> bool:
        """The similarity label (bottom 2) is never forced.  reference: include/caffe/loss_layers.hpp:170-172."""
        return bottom != 2

    def forward(self, a, b, sim):
        return (ops.reference.contrastive_loss(a, b, sim, self.margin),)


@register("ACCURACY")
class AccuracyLayer(Layer):
    """reference: src/caffe/layers/accuracy_layer.cpp:14-66 (top-k, not differentiable)."""
    exact_bottoms = 2
    exact_tops = 1

    def setup(self, bottom_shapes):
        self.top_k = int(self.lp.accuracy_param.top_k)
        n, c, h, w = bottom_shapes[0]
        if self.top_k > c * h * w:
            raise ValueError("top_k must be less than or equal to the number of classes.")
        return [(1, 1, 1, 1)]

    @torch.no_grad()
    def forward(self, x, label):
        return (ops.reference.accuracy(x, label, self.top_k),)
