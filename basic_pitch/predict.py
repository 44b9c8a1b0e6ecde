"""Drop-in for reference: basic_pitch/predict.py (the `basic-pitch` console entry point): `python -m basic_pitch.predict`
forwards to the command line of basic_pitch_b200 (same flags)."""
from basic_pitch_b200.predict import main  # noqa: F401

if __name__ == "__main__":
    main()
