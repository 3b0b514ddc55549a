"""GPU probe of the device building blocks (test infrastructure): pdq_probe.cu, built by build.py, driven by probe.py."""
