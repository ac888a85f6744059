"""Mirror of the reference's ``NPHM.evaluation`` package for the part that is data-parallel (SURVEY.md 8f-4): ``metrics``, and the
surface sampling of the evaluation protocol, ``render_utils`` (native depth / normal rendering) and ``sampling`` (eval.py)."""
