"""CPU oracle for the Local-Hints-Network forward path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``oracle/`` is imported by the product
package (``interactive_deep_colorization_b200``).  Allowed importers: ``tests/``,
``__graft_entry__.smoke()`` and the ``cpu_baseline`` / ``--impl reference`` legs of
``bench.py`` -- and there only as the checker / the timed CPU baseline.

Parity pin status (see DESIGN.md "Oracle"):
  * network trunk + regression head + 529-bin dist head (rows a3..a9, a12, a13 of
    SURVEY.md section 8a): PINNED against the unmodified reference
    ``models/pytorch/model.py`` (outputs stored as golden
    vectors + generating script live in ``tests/golden/``.
  * Lab<->RGB (rows a10, a11): restatement of scikit-image 0.13 ``color.rgb2lab /
    lab2rgb`` (absent from the image, not vendored by the reference): PARITY UNPINNED
    by any reference test; pinned only by our own golden vectors.
  * Caffe-spec 313-bin head / annealed mean / global-hints branch (rows a14, a15):
    no Caffe runtime, no reference test vectors: PARITY UNPINNED.
"""
