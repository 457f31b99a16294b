"""Operator layer: routing, sparse dispatch/combine, grouped expert GEMMs (native sm_90a kernels + CPU paths)."""
