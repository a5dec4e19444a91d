"""TEST INFRASTRUCTURE ONLY — minimal CPU restatement of the `diffusers==0.19.3` symbols
(requirements.txt:2 of the reference; source NOT under the reference checkout) that the reference's
model files import.  Written from the published behaviour of diffusers 0.19.3; "parity unpinned"
against a real diffusers install (none is available offline).  Used only by oracle/ref_loader.py
to import the reference's own model files unmodified from a checkout of the reference.
"""
__version__ = "0.19.3-stub"
