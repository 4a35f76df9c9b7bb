"""Import shim for the reference's `matplotlib`: only `import matplotlib.pyplot as plt` is needed, because every
plt.imsave call in the reference's visualisation sits under `if False`."""
