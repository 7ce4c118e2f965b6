"""Segment Anything (registered on import: ``import tfimm.architectures.segment_anything``, as in the reference, whose
package ``__init__`` does not import it either)."""
from .sam import *  # noqa: F401,F403
