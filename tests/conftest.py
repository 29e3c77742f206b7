import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))

def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA GPU, an H100 (sm_90a); select with -m gpu")
