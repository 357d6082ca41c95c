"""Drop-in replacement of the reference's top-level ``inference`` package
(the reference's inference/__init__.py:1-8).  Put this repository ahead of the reference on
``sys.path`` / ``PYTHONPATH`` and ``infer.py``, ``batch_infer.py`` and ``webui.py`` resolve
``inference.MIDIExtractionInference`` / ``inference.QuantizedMIDIExtractionInference`` to the
H100-native implementation (some_b200.plugin) without any change (see INTEGRATION.md)."""
from some_b200.plugin import (BaseInference, MIDIExtractionInference, QuantizedMIDIExtractionInference,
                              task_inference_mapping)

__all__ = ['BaseInference', 'MIDIExtractionInference', 'QuantizedMIDIExtractionInference',
           'task_inference_mapping']
