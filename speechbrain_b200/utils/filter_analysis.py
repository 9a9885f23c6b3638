"""Filter properties -- mirror of speechbrain.utils.filter_analysis (FilterProperties, stack_filter_properties) and of
``upalign_value`` (speechbrain/lobes/features.py:484-493): how window size, stride, dilation and causality combine when
filters are stacked.  ``StreamingFeatureWrapper`` derives its padding from them.  Host-side arithmetic only."""
from dataclasses import dataclass


def upalign_value(x, to: int) -> int:
    """``x`` rounded up to a multiple of ``to``."""
    assert x >= 0
    if (x % to) == 0:
        return x
    return x + to - (x % to)


@dataclass
class FilterProperties:
    """Properties of something that behaves like a filter over time: ``window_size`` input frames per output frame,
    ``stride`` input frames between consecutive outputs, ``dilation`` (1: none), ``causal``."""

    window_size: int
    stride: int = 1
    dilation: int = 1
    causal: bool = False

    def __post_init__(self):
        assert self.window_size > 0
        assert self.stride > 0
        assert self.dilation > 0, "Dilation must be >0. NOTE: a dilation of 1 means no dilation."

    @staticmethod
    def pointwise_filter() -> "FilterProperties":
        return FilterProperties(window_size=1, stride=1)

    def get_effective_size(self):
        """Input frames the window spans, including those skipped by dilation."""
        return 1 + ((self.window_size - 1) * self.dilation)

    def get_convolution_padding(self):
        """Frames to insert on each end for a typical convolution."""
        if self.window_size % 2 == 0:
            raise ValueError("Cannot determine padding with even window size")
        if self.causal:
            return self.get_effective_size() - 1
        return (self.get_effective_size() - 1) // 2

    def get_noncausal_equivalent(self):
        """A non-causal filter whose outputs depend on the same input frames (plus some false dependencies)."""
        if not self.causal:
            return self
        return FilterProperties(window_size=(self.window_size - 1) * 2 + 1, stride=self.stride, dilation=self.dilation,
                                causal=False)

    def with_on_top(self, other, allow_approximate=True):
        """The properties of ``other(self(x))``.  With ``allow_approximate`` an even window is widened by one and a mix of
        causal and non-causal filters is made non-causal, instead of raising."""
        self_size = self.window_size
        if other.window_size % 2 == 0:
            if allow_approximate:
                other_size = other.window_size + 1
            else:
                raise ValueError("The filter to append cannot have an uneven window size. Specify `allow_approximate=True` "
                                 "if you do not need to analyze exact dependencies.")
        else:
            other_size = other.window_size
        if (self.causal or other.causal) and not (self.causal and other.causal):
            if allow_approximate:
                return self.get_noncausal_equivalent().with_on_top(other.get_noncausal_equivalent())
            raise ValueError("Cannot express exact properties of causal and non-causal filters. Specify "
                             "`allow_approximate=True` if you do not need to analyze exact dependencies.")
        out_size = self_size + (self.stride * (other_size - 1))
        return FilterProperties(out_size, self.stride * other.stride, self.dilation * other.dilation, self.causal)


def stack_filter_properties(filters, allow_approximate=True):
    """The properties of ``filters`` stacked in order (``[a, b, c]`` models ``c(b(a(x)))``); an item that is not a
    ``FilterProperties`` gives its ``get_filter_properties()``.  An empty sequence is the pointwise filter."""
    ret = FilterProperties.pointwise_filter()
    for prop in filters:
        if not isinstance(prop, FilterProperties):
            prop = prop.get_filter_properties()
        ret = ret.with_on_top(prop, allow_approximate)
    return ret
