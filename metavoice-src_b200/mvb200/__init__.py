"""mvb200: H100-native engine behind MetaVoice-1B's TTS.synthesise() hot path (see DESIGN.md)."""
