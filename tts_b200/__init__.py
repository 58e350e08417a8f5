"""tts_b200 -- H100-native (sm_90a) VITS + HiFiGAN inference hot path behind the coqui-ai/TTS
operator API.  See DESIGN.md / INTEGRATION.md."""
__version__ = "0.1.0"
