"""The reference's package name over the GPU engine; see compat/README.md."""
