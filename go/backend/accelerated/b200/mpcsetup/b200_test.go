//go:build b200

package mpcsetup_test

import (
	"bytes"
	"testing"

	"github.com/consensys/gnark-crypto/ecc"
	cmpc "github.com/consensys/gnark-crypto/ecc/bn254/mpcsetup"
	"github.com/consensys/gnark/backend/groth16"
	"github.com/consensys/gnark/backend/groth16/bn254/mpcsetup"
	cs "github.com/consensys/gnark/constraint/bn254"
	"github.com/consensys/gnark/frontend"
	"github.com/consensys/gnark/frontend/cs/r1cs"

	b200mpc "github.com/consensys/gnark/backend/accelerated/b200/mpcsetup/bn254"
)

type cubic struct {
	X frontend.Variable
	Y frontend.Variable `gnark:",public"`
}

func (c *cubic) Define(api frontend.API) error {
	x3 := api.Mul(c.X, c.X, c.X)
	api.AssertIsEqual(c.Y, api.Add(x3, c.X, 5))
	return nil
}

// committedCubic adds a BSB22 commitment to X and Y, so that the key has one SigmaCKK / G2.Sigma pair
type committedCubic struct {
	X frontend.Variable
	Y frontend.Variable `gnark:",public"`
}

func (c *committedCubic) Define(api frontend.API) error {
	x3 := api.Mul(c.X, c.X, c.X)
	api.AssertIsEqual(c.Y, api.Add(x3, c.X, 5))
	cm, err := api.(frontend.Committer).Commit(c.X, c.Y)
	if err != nil {
		return err
	}
	api.AssertIsDifferent(cm, 0)
	return nil
}

// The mirror of gnark's mpcsetup TestAll: three phase-1 and three phase-2 contributions made on the device, a chain
// that gnark's own VerifyPhase1 and VerifyPhase2 must accept, and a proof with the resulting key that verifies; once
// without a commitment and once with one (SigmaCKK and G2.Sigma updated by ContributePhase2).
func TestContributionsBN254(t *testing.T) {
	t.Run("plain", func(t *testing.T) { testChain(t, &cubic{}, &cubic{X: 3, Y: 35}) })
	t.Run("commitment", func(t *testing.T) { testChain(t, &committedCubic{}, &committedCubic{X: 3, Y: 35}) })
}

func testChain(t *testing.T, circuit, assignment frontend.Circuit) {
	ccs, err := frontend.Compile(ecc.BN254.ScalarField(), r1cs.NewBuilder, circuit)
	if err != nil {
		t.Fatal(err)
	}
	domainSize := ecc.NextPowerOfTwo(uint64(ccs.GetNbConstraints()))

	var bb bytes.Buffer
	if _, err := mpcsetup.NewPhase1(domainSize).WriteTo(&bb); err != nil {
		t.Fatal(err)
	}
	phase1 := make([]*mpcsetup.Phase1, 3)
	for i := range phase1 {
		var next bytes.Buffer
		if err := b200mpc.ContributePhase1(bytes.NewReader(bb.Bytes()), &next); err != nil {
			t.Fatal(err)
		}
		phase1[i] = new(mpcsetup.Phase1)
		if n, err := phase1[i].ReadFrom(bytes.NewReader(next.Bytes())); err != nil || int(n) != next.Len() {
			t.Fatalf("contribution %d: read %d of %d bytes: %v", i, n, next.Len(), err)
		}
		bb = next
	}
	commons, err := mpcsetup.VerifyPhase1(domainSize, []byte("testing phase1"), phase1...)
	if err != nil {
		t.Fatal(err)
	}

	r1csImpl := ccs.(*cs.R1CS)
	// a Phase2 object that fails must be left as it was: a mismatched commitment count is refused before any change
	{
		var bad mpcsetup.Phase2
		bad.Initialize(r1csImpl, &commons)
		bad.Sigmas = append(bad.Sigmas, cmpc.UpdateProof{})
		var before bytes.Buffer
		if _, err := bad.WriteTo(&before); err != nil {
			t.Fatal(err)
		}
		if err := b200mpc.ContributePhase2(&bad); err == nil {
			t.Fatal("mismatched commitment counts accepted")
		}
		var after bytes.Buffer
		if _, err := bad.WriteTo(&after); err != nil {
			t.Fatal(err)
		}
		if !bytes.Equal(before.Bytes(), after.Bytes()) {
			t.Fatal("a refused contribution changed its Phase2")
		}
	}
	var p2 mpcsetup.Phase2
	p2.Initialize(r1csImpl, &commons)
	phase2 := make([]*mpcsetup.Phase2, 3)
	for i := range phase2 {
		if err := b200mpc.ContributePhase2(&p2); err != nil {
			t.Fatal(err)
		}
		bb.Reset()
		if _, err := p2.WriteTo(&bb); err != nil {
			t.Fatal(err)
		}
		phase2[i] = new(mpcsetup.Phase2)
		if _, err := phase2[i].ReadFrom(bytes.NewReader(bb.Bytes())); err != nil {
			t.Fatal(err)
		}
	}
	pk, vk, err := mpcsetup.VerifyPhase2(r1csImpl, &commons, []byte("testing phase2"), phase2...)
	if err != nil {
		t.Fatal(err)
	}

	w, err := frontend.NewWitness(assignment, ecc.BN254.ScalarField())
	if err != nil {
		t.Fatal(err)
	}
	proof, err := groth16.Prove(ccs, pk, w)
	if err != nil {
		t.Fatal(err)
	}
	pub, err := w.Public()
	if err != nil {
		t.Fatal(err)
	}
	if err := groth16.Verify(proof, vk, pub); err != nil {
		t.Fatal(err)
	}
}
