"""CPU oracle for the openrec.tf2 training hot path -- TEST INFRASTRUCTURE ONLY.

Nothing under ``oracle/`` is part of the product.  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference``
legs may import it, and only as the checker (or as the timed CPU arm).

PARITY UNPINNED (TensorFlow part): the arithmetic of the reference path lives in
TensorFlow/Keras (only pin: ``docs_requirements.txt:2`` ``tensorflow==2.0.1``), which
is neither vendored in the reference nor installable here, and the reference has
no tests / golden vectors.  What *is* pinned: the reference's own Python composition
(``openrec/tf2/{modules,recommenders,metrics}``) executed verbatim under a torch-backed
``tensorflow`` stand-in (``tests/golden/make_golden.py``) -> fixtures in
``tests/golden/*.npz``; and the reference's sampler code run directly.
"""
