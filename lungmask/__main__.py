"""`python -m lungmask INPUT OUTPUT` -> the H100 engine's CLI."""
from lungmask_b200.__main__ import main

if __name__ == "__main__":
    main()
