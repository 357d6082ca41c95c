"""some_b200 — SOME's inference hot path on H100 (sm_90a).

Public surface (nothing is imported eagerly; the CUDA library is loaded on first use and there is no CPU fallback):

* ``some_b200.plugin``  — ``BaseInference`` / ``MIDIExtractionInference`` / ``QuantizedMIDIExtractionInference``
  (the reference's plugin classes; also importable as the top-level ``inference`` package)
* ``some_b200.engine``  — ``Engine`` (``infer``, ``infer_sliced``, ``enqueue``), ``pinned_array``
* ``some_b200.dist``    — ``infer_sharded`` / ``infer_sliced_sharded`` (one process per GPU, one all-gather of notes)
* ``some_b200.slicer``  — ``Slicer`` (drop-in for ``utils.slicer2.Slicer``, RMS on the GPU)
* ``some_b200.midi``    — ``build_midi_file`` (dependency-free SMF writer)
* ``some_b200.batch``   — ``transcribe_recordings`` / ``batch_infer_dataset`` (dataset-level driver)
* ``some_b200._lib``    — ctypes binding of ``include/some_b200.h``
"""
