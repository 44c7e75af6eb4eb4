"""Drop-in for the reference's `gcn_lib` package (same sub-packages, class names,
constructor / forward signatures and state_dict keys; SURVEY.md 8b), with the
message-passing arithmetic running in the sm_90a kernels of libdgcn.so."""
