"""Classifier guidance without PyTorch autograd: ``make_cond_fn(classifier, scale)`` is the reference's ``cond_fn``
(diffusion.py:183-189) over a ``ddnm_b200.model.EncoderUNetModel``.

    classifier = create_classifier(**args_to_dict(config.classifier, classifier_defaults().keys()))
    classifier.load_state_dict(ckpt)
    cls_fn = make_cond_fn(classifier, config.classifier.classifier_scale)
    ddnm_diffusion(..., cls_fn=cls_fn)     # the sampler runs the gradient inside the library, no Python callback

Called from Python, ``cls_fn(x, t, y)`` returns the gradient as a CUDA tensor, so it also works wherever a Python cond_fn is
accepted (``hq.restore``)."""
from .model import EncoderUNetModel


class ClassifierCondFn:
    """cond_fn(x, t, y) = classifier_scale * d/dx sum_b log_softmax(classifier(x, t))[b, y_b]."""

    def __init__(self, classifier, classifier_scale):
        if not isinstance(classifier, EncoderUNetModel):
            raise TypeError("make_cond_fn needs a ddnm_b200.model.EncoderUNetModel (create_classifier)")
        self.classifier = classifier
        self.scale = float(classifier_scale)

    def __call__(self, x, t, y):
        return self.classifier.grad(x.float(), t, y, self.scale)


def make_cond_fn(classifier, classifier_scale):
    return ClassifierCondFn(getattr(classifier, "module", classifier), classifier_scale)
